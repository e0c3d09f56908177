"""magicpig_b200 -- H100-native LSH-sampled sparse-attention decode path (drop-in for MagicPIG's
`models/attnserver.py` operator surface).  See DESIGN.md and include/magicpig_b200.h.

Layout:  csrc/ (sm_90a kernels + C ABI)  _native.py (ctypes)  ops.py (Context, LSH,
SparseAttentionServer mirrors)  attnserver.py (LSHSparseAttnServer)  synth.py (seeded inputs)
"""
__version__ = "0.1.0"

from ._native import MagicPigError  # noqa: F401


def __getattr__(name):
    # lazy: importing the package must not require the CUDA library (CPU-only tooling, build step)
    if name in ("Context", "LSH", "SparseAttentionServer"):
        from . import ops
        return getattr(ops, name)
    if name == "LSHSparseAttnServer":
        from .attnserver import LSHSparseAttnServer
        return LSHSparseAttnServer
    raise AttributeError(name)
