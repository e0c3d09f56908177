"""Build the UNMODIFIED reference CPU operators into oracle/_ref/  (TEST INFRASTRUCTURE ONLY).

This compiles MagicPIG's own `library/lsh` and `library/sparse_attention` pybind modules
straight from the sources where they lie in a checkout of the reference (`MAGICPIG_REFERENCE`;
nothing is copied into this repository) and drops only the resulting shared objects under
`oracle/_ref/` (git-ignored build products; a machine without the reference can use prebuilt ones).

It mirrors the reference's own build lines:
  * library/lsh/setup.py:5-13                ->  oracle/_ref/lsh.so
  * library/sparse_attention/setup.py:33-51  ->  oracle/_ref/{bf16,f32}/sparse_attention_cpu.so
    (two flavours: `-mavx512bf16` as the reference auto-selects on a BF16-capable host,
    and the plain AVX512F build for hosts without AVX512_BF16 -- the loader in
    `oracle/ref_loader.py` picks the one the running CPU supports.)

Only `tests/`, `__graft_entry__.smoke()`, `__graft_entry__.build()` and `bench.py`'s CPU
baseline / `--impl reference` legs may use the result.  The product path never does.

Run:  python oracle/build_ref.py            (needs the reference checkout; ~2-3 min)
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import sysconfig
import time

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
REF = os.environ.get("MAGICPIG_REFERENCE", "/root/reference")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"  # /opt/gcc wrapper lacks libgomp.spec


def _torch_flags():
    import torch
    from torch.utils import cpp_extension as ce

    inc = []
    for p in ce.include_paths():
        inc += ["-isystem", p]
    inc += ["-isystem", sysconfig.get_paths()["include"]]
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    defs = [
        "-DTORCH_API_INCLUDE_EXTENSION_H",
        f"-D_GLIBCXX_USE_CXX11_ABI={abi}",  # reference pins 0 (torch 2.3); match the torch we link against
        "-DNDEBUG",  # the reference's setuptools build inherits -DNDEBUG (asserts compiled out)
    ]
    link = [f"-L{libdir}", "-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", f"-Wl,-rpath,{libdir}"]
    return inc, defs, link


def _compile(name: str, sources: list[str], extra_inc: list[str], extra_flags: list[str], out_so: str):
    inc, defs, link = _torch_flags()
    os.makedirs(os.path.dirname(out_so), exist_ok=True)
    objdir = os.path.join(OUT, "obj", name + "_" + os.path.basename(os.path.dirname(out_so)))
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src in sources:
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        objs.append(obj)
        cmd = [CXX, "-c", src, "-o", obj, "-fPIC", "-O3", "-std=c++17", "-fopenmp", "-mavx512f",
               f"-DTORCH_EXTENSION_NAME={name}", *defs, *extra_flags, *inc]
        for p in extra_inc:
            cmd += ["-I", p]
        procs.append((src, subprocess.Popen(cmd)))
    for src, p in procs:
        if p.wait() != 0:
            raise RuntimeError(f"compile failed: {src}")
    cmd = [CXX, "-shared", "-o", out_so, *objs, "-fopenmp", *link]
    subprocess.check_call(cmd)


def build(force: bool = False) -> bool:
    """Returns True if oracle/_ref is populated (built now or already present)."""
    lsh_so = os.path.join(OUT, "lsh.so")
    sa_bf16 = os.path.join(OUT, "bf16", "sparse_attention_cpu.so")
    sa_f32 = os.path.join(OUT, "f32", "sparse_attention_cpu.so")
    have = all(os.path.exists(p) for p in (lsh_so, sa_bf16, sa_f32))
    if have and not force:
        return True
    if not os.path.isdir(os.path.join(REF, "library", "lsh")):
        # no reference checkout here -> only prebuilt files can be used
        return have
    t0 = time.time()
    lsh_dir = os.path.join(REF, "library", "lsh")
    sa_dir = os.path.join(REF, "library", "sparse_attention")
    fb = os.path.join(sa_dir, "3rdparty", "FBGEMM")
    _compile("lsh", [os.path.join(lsh_dir, "lsh.cc")], [lsh_dir], [], lsh_so)
    sa_src = [os.path.join(sa_dir, "sparse_attention.cc")] + [
        os.path.join(fb, "src", f)
        for f in ("FbgemmBfloat16Convert.cc", "FbgemmBfloat16ConvertAvx2.cc",
                  "FbgemmBfloat16ConvertAvx512.cc", "RefImplementations.cc", "Utils.cc")
    ]
    sa_inc = [sa_dir, os.path.join(fb, "include")]
    _compile("sparse_attention_cpu", sa_src, sa_inc, ["-mavx512bf16"], sa_bf16)
    _compile("sparse_attention_cpu", sa_src, sa_inc, [], sa_f32)
    shutil.rmtree(os.path.join(OUT, "obj"), ignore_errors=True)
    print(f"[oracle/_ref] built lsh + sparse_attention_cpu (bf16, f32) in {time.time() - t0:.0f}s", file=sys.stderr)
    return True


if __name__ == "__main__":
    ok = build(force="--force" in sys.argv)
    print("oracle/_ref:", "ready" if ok else "unavailable (no reference checkout and no prebuilt files)")
