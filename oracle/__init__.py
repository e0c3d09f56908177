"""oracle -- CPU parity checker for the LSH sparse-attention decode path.  TEST INFRASTRUCTURE ONLY.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s `cpu_baseline` / `--impl reference`
legs may import this package.  The product (`magicpig_b200`) never does and has no CPU
fallback: it raises if the CUDA library is missing.

Two checkers live here:
  * `oracle.port`  (this module): ctypes front-end of `mpig_oracle.c`, the plain-C restatement
    of the reference algorithm (each C function cites the reference file:line it follows).
  * `oracle.ref_loader`: the UNMODIFIED reference operators (`lsh.LSH`,
    `sparse_attention_cpu.SparseAttentionServer`) compiled from a checkout of the reference by
    `oracle/build_ref.py` into `oracle/_ref/`.

Parity status: pinned (see header of mpig_oracle.c and tests/test_oracle_cpu.py).
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = os.path.join(_HERE, "_build")
_SO = os.path.join(_BUILD, "libmpig_oracle.so")
_SRC = os.path.join(_HERE, "mpig_oracle.c")
_lib = None


def build(force: bool = False) -> str:
    """gcc the C restatement into oracle/_build/ (git-ignored build product)."""
    if force or (not os.path.exists(_SO)) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        os.makedirs(_BUILD, exist_ok=True)
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.check_call([cc, "-O2", "-fPIC", "-shared", "-o", _SO, _SRC, "-lm"])
    return _SO


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
        _lib.orc_f32_to_bf16_half_up.restype = ctypes.c_uint16
        _lib.orc_f32_to_bf16_half_up.argtypes = [ctypes.c_float]
        _lib.orc_f32_to_bf16_rne.restype = ctypes.c_uint16
        _lib.orc_f32_to_bf16_rne.argtypes = [ctypes.c_float]
    return _lib


def _p(t: torch.Tensor | None):
    if t is None:
        return ctypes.c_void_p(0)
    assert t.device.type == "cpu" and t.is_contiguous(), "oracle takes contiguous CPU tensors"
    return ctypes.c_void_p(t.data_ptr())


# ---------------------------------------------------------------- stage 1
def simhash(q_bf16: torch.Tensor, hash_func_bf16: torch.Tensor, K: int, L: int):
    """codes (H, L) int32 and min |projection| per code (H, L) fp32.  models/attnserver.py:264-270."""
    assert q_bf16.dtype == torch.bfloat16 and hash_func_bf16.dtype == torch.bfloat16
    H, d = q_bf16.shape
    assert hash_func_bf16.shape == (d, K * L)
    codes = torch.zeros((H, L), dtype=torch.int32)
    margin = torch.zeros((H, L), dtype=torch.float32)
    lib().orc_simhash(_p(q_bf16.contiguous()), _p(hash_func_bf16.contiguous()), H, d, K, L, _p(codes), _p(margin))
    return codes, margin


# ---------------------------------------------------------------- tables + stage 2
class Tables:
    """Reference-layout hash tables of ONE (layer, request): lsh.cc:44-91 members."""

    def __init__(self, Hkv: int, L: int, K: int, max_length: int):
        self.Hkv, self.L, self.K, self.NB, self.max_length = Hkv, L, K, 1 << K, max_length
        self.start = torch.zeros((Hkv, L, self.NB), dtype=torch.int32)
        self.end = torch.zeros((Hkv, L, self.NB), dtype=torch.int32)
        self.table = torch.zeros((Hkv, L, max_length), dtype=torch.int32)
        self.n = 0

    def fill(self, sorted_codes: torch.Tensor, sorted_indices: torch.Tensor):
        """LSH::fill, lsh.cc:143-201.  sorted_codes int16 (Hkv,L,n), sorted_indices int32 (Hkv,L,n)."""
        assert sorted_codes.dtype == torch.int16 and sorted_indices.dtype == torch.int32
        Hkv, L, n = sorted_codes.shape
        assert (Hkv, L) == (self.Hkv, self.L) and n <= self.max_length
        self.n = n
        lib().orc_lsh_fill(_p(sorted_codes.contiguous()), _p(sorted_indices.contiguous()), Hkv, L, n, self.NB,
                           self.max_length, _p(self.start), _p(self.end), _p(self.table))


def batch_retrieve(tables: Tables, query: torch.Tensor, G: int):
    """LSH::batch_retrieve for ONE request (lsh.cc:210-288).  query int32 (Hkv*G, L).
    Returns results (H, max_length) int32 [first nnz valid, second-hit order], nnz (H,), mask uint8 (H, max_length)."""
    H = query.shape[0]
    assert query.dtype == torch.int32 and query.shape[1] == tables.L and H == tables.Hkv * G
    results = torch.zeros((H, tables.max_length), dtype=torch.int32)
    nnz = torch.zeros((H,), dtype=torch.int32)
    mask = torch.zeros((H, tables.max_length), dtype=torch.uint8)
    lib().orc_lsh_batch_retrieve(_p(tables.start), _p(tables.end), _p(tables.table), tables.L, tables.NB,
                                 tables.max_length, G, H, _p(query.contiguous()), _p(results), _p(nnz), _p(mask))
    return results, nnz, mask


def collision_counts(key_codes: torch.Tensor, query: torch.Tensor, G: int) -> torch.Tensor:
    """Full collision counts (H, n) straight from unsorted key codes int16 (Hkv, L, n): lsh/test.py:43."""
    Hkv, L, n = key_codes.shape
    H = query.shape[0]
    assert key_codes.dtype == torch.int16 and query.dtype == torch.int32 and H == Hkv * G
    counts = torch.zeros((H, n), dtype=torch.int32)
    lib().orc_collision_counts(_p(key_codes.contiguous()), L, n, G, H, _p(query.contiguous()), _p(counts))
    return counts


# ---------------------------------------------------------------- stage 3
def attention_wrapper(key: torch.Tensor, value: torch.Tensor, key_norm: torch.Tensor, K: int, L: int,
                      query: torch.Tensor, query_norm: torch.Tensor, ind: torch.Tensor, nnz: torch.Tensor,
                      want_score: bool = False):
    """SparseAttentionServer::attention_wrapper (sparse_attention.cc:629-745, 867-925).
    key/value bf16 (B*Hkv, max_length, d); key_norm fp32 (B*Hkv, max_length); query bf16 (H, d);
    query_norm fp32 (H,); ind int32 (H, max_length); nnz int32 (H,).
    Returns output bf16 (H, d), max_value_expsum fp32 (2, H) [row1 = base-2 LSE], score or None."""
    BHkv, max_length, d = key.shape
    H = query.shape[0]
    G = H // BHkv
    assert key.dtype == torch.bfloat16 and value.dtype == torch.bfloat16 and query.dtype == torch.bfloat16
    assert key_norm.dtype == torch.float32 and query_norm.dtype == torch.float32
    assert ind.dtype == torch.int32 and nnz.dtype == torch.int32 and ind.shape == (H, max_length)
    out = torch.zeros((H, d), dtype=torch.bfloat16)
    mve = torch.zeros((2, H), dtype=torch.float32)
    score = torch.zeros((H, max_length), dtype=torch.float32) if want_score else None
    lib().orc_attention_wrapper(_p(key.contiguous()), _p(value.contiguous()), _p(key_norm.contiguous()), d, max_length,
                                G, H, K, L, _p(query.contiguous()), _p(query_norm.contiguous()), _p(ind.contiguous()),
                                _p(nnz.contiguous()), _p(out), _p(mve), _p(score))
    return out, mve, score


def window_attention(key: torch.Tensor, value: torch.Tensor, query: torch.Tensor, G: int):
    """Plain attention of each q-head over its kv-group's contiguous window.
    key/value bf16 (BHkv, len, d), query bf16 (H, d).  Returns out fp32 (H, d), lse2 fp32 (H,)."""
    BHkv, ln, d = key.shape
    H = query.shape[0]
    out = torch.zeros((H, d), dtype=torch.float32)
    lse = torch.zeros((H,), dtype=torch.float32)
    key, value, query = key.contiguous(), value.contiguous(), query.contiguous()
    for h in range(H):
        g = h // G
        lib().orc_window_attention_head(ctypes.c_void_p(key[g].data_ptr()), ctypes.c_void_p(value[g].data_ptr()), d, ln,
                                        ctypes.c_void_p(query[h].data_ptr()), ctypes.c_void_p(out[h].data_ptr()),
                                        ctypes.c_void_p(lse[h:].data_ptr()))
    return out, lse


def merge_state(o_a: torch.Tensor, lse_a: torch.Tensor, o_b: torch.Tensor, lse_b: torch.Tensor):
    """flashinfer.merge_state restated (base-2 LSE).  o_* fp32 (H, d), lse_* fp32 (H,)."""
    H, d = o_a.shape
    o = torch.zeros((H, d), dtype=torch.float32)
    lse = torch.zeros((H,), dtype=torch.float32)
    o_a, o_b = o_a.float().contiguous(), o_b.float().contiguous()
    for h in range(H):
        lib().orc_merge_state(ctypes.c_void_p(o_a[h].data_ptr()), ctypes.c_float(float(lse_a[h])),
                              ctypes.c_void_p(o_b[h].data_ptr()), ctypes.c_float(float(lse_b[h])), d,
                              ctypes.c_void_p(o[h].data_ptr()), ctypes.c_void_p(lse[h:].data_ptr()))
    return o, lse
