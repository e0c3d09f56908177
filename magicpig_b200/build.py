"""Build the sm_90a (H100) CUDA library in-tree:  magicpig_b200/lib/libmagicpig_b200.so

nvcc cross-compiles without a GPU.  The .so and its objects are build products (git-ignored).
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libmagicpig_b200.so")
SOURCES = ["context.cu", "tables.cu", "store.cu", "fused.cu", "attend_mma.cu", "attend_dense.cu", "attend_chunk.cu", "attend_prefill.cu", "simhash.cu", "step.cu", "decode.cu", "peer.cu", "aux_ops.cu", "aux_gemv.cu", "aux_sample.cu", "keyhash.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"]


def _newest_input() -> float:
    t = os.path.getmtime(os.path.abspath(__file__))   # the flags (target architecture) live here
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(root):
            t = max(t, os.path.getmtime(os.path.join(root, f)))
    return t


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _newest_input():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    extra = ["-Xptxas", "-v"] if verbose else []

    def cc(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [NVCC, *FLAGS, *extra, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, obj, r

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        results = list(ex.map(cc, SOURCES))
    objs = []
    for src, obj, r in results:
        if verbose or r.returncode != 0:
            sys.stderr.write(f"---- {src}\n{r.stdout}{r.stderr}\n")
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}")
        objs.append(obj)
    cmd = [NVCC, "-shared", "-o", LIB, *objs, "-cudart", "shared", "-ccbin", FLAGS[-1]]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
