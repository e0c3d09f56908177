"""Load the UNMODIFIED reference operators from oracle/_ref/ (TEST INFRASTRUCTURE ONLY).

`lsh.LSH` (library/lsh/lsh.cc:316-326) and `sparse_attention_cpu.SparseAttentionServer`
(library/sparse_attention/sparse_attention.cc:1243-1263) are compiled from a checkout of the
reference by `oracle/build_ref.py`.  Two flavours of sparse_attention_cpu exist; the loader picks the
AVX512_BF16 one only when the running CPU has that extension (it would SIGILL otherwise).
"""
from __future__ import annotations

import importlib.util
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF = os.path.join(_HERE, "_ref")
_cache: dict = {}


def cpu_flags() -> set[str]:
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("flags"):
                    return set(line.split(":", 1)[1].split())
    except OSError:
        pass
    return set()


def flavour() -> str:
    return "bf16" if "avx512_bf16" in cpu_flags() else "f32"


def available() -> bool:
    if "avx512f" not in cpu_flags():
        return False
    return os.path.exists(os.path.join(_REF, "lsh.so")) and os.path.exists(
        os.path.join(_REF, flavour(), "sparse_attention_cpu.so"))


def _load(name: str, path: str):
    import torch  # noqa: F401  (libtorch must be loaded before the extension)

    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    # the reference modules print / run nothing at import; keep them out of sys.modules' way
    sys.modules.setdefault("_mpig_ref_" + name, mod)
    spec.loader.exec_module(mod)
    return mod


def load():
    """Returns (lsh_module, sparse_attention_cpu_module, flavour).  Raises if unavailable."""
    if "mods" not in _cache:
        if not available():
            raise RuntimeError("oracle/_ref not built (run `python oracle/build_ref.py` where the reference is checked out) "
                               "or CPU lacks AVX-512F")
        fl = flavour()
        _cache["mods"] = (_load("lsh", os.path.join(_REF, "lsh.so")),
                          _load("sparse_attention_cpu", os.path.join(_REF, fl, "sparse_attention_cpu.so")), fl)
    return _cache["mods"]
