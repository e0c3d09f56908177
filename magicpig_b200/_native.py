"""ctypes binding of libmagicpig_b200.so (the C ABI declared in include/magicpig_b200.h).

No torch types cross the boundary: tensors are passed as raw device pointers + the current CUDA
stream handle.  There is no CPU fallback: if the library is missing this raises, loudly.
"""
from __future__ import annotations

import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libmagicpig_b200.so")
HEADER_PATH = os.path.join(_HERE, "..", "include", "magicpig_b200.h")

MPIG_ABI_VERSION = 1
MPIG_OK = 0


class MpigConfig(ctypes.Structure):
    _fields_ = [
        ("abi_version", ctypes.c_int32),
        ("device", ctypes.c_int32),
        ("K", ctypes.c_int32),
        ("L", ctypes.c_int32),
        ("num_layers", ctypes.c_int32),
        ("num_attention_heads", ctypes.c_int32),
        ("num_key_value_heads", ctypes.c_int32),
        ("head_dim", ctypes.c_int32),
        ("batch_size", ctypes.c_int32),
        ("max_length", ctypes.c_int32),
        ("num_sink_tokens", ctypes.c_int32),
        ("num_local_tokens", ctypes.c_int32),
        ("generation_buffer", ctypes.c_int32),
        ("num_dense_layers", ctypes.c_int32),
        ("dense_layers", ctypes.c_int32 * 16),
        ("alloc_dense_kv", ctypes.c_int32),
        ("ctas_per_sm", ctypes.c_int32),
        ("num_contexts", ctypes.c_int32),
        ("dense_tail_rows", ctypes.c_int32),
        ("shared_spill", ctypes.c_int32),
        ("reserved", ctypes.c_int32 * 4),
    ]


class MpigSampleFilters(ctypes.Structure):
    """mpig_sample_filters (include/magicpig_b200_aux.h): five per-request device arrays and the penalty table."""
    _fields_ = [
        ("top_k", ctypes.c_void_p),
        ("min_p", ctypes.c_void_p),
        ("repetition_penalty", ctypes.c_void_p),
        ("presence_penalty", ctypes.c_void_p),
        ("frequency_penalty", ctypes.c_void_p),
        ("table", ctypes.c_void_p),
        ("ld", ctypes.c_int64),
    ]


class MagicPigError(RuntimeError):
    pass


_lib = None
_vp = ctypes.c_void_p
_i = ctypes.c_int

# name -> (restype, argtypes)
_SIGNATURES = {
    "mpig_create": (_i, [ctypes.POINTER(MpigConfig), ctypes.POINTER(_vp)]),
    "mpig_destroy": (None, [_vp]),
    "mpig_last_error": (ctypes.c_char_p, []),
    "mpig_abi_version": (_i, []),
    "mpig_device_bytes": (ctypes.c_size_t, [_vp]),
    "mpig_set_option": (_i, [_vp, ctypes.c_char_p, ctypes.c_int64]),
    "mpig_clear": (_i, [_vp, _vp]),
    "mpig_set_hash_func": (_i, [_vp, _vp, _vp]),
    "mpig_lsh_fill": (_i, [_vp, _i, _i, _vp, _vp, _i, _vp]),
    "mpig_hash_keys": (_i, [_vp, _vp, _i, _vp, _vp]),
    "mpig_lsh_build": (_i, [_vp, _i, _i, _vp, _i, _vp]),
    "mpig_lsh_batch_retrieve": (_i, [_vp, _i, _vp, _vp, _vp, _vp]),
    "mpig_lsh_get_mask": (_i, [_vp, _vp, _vp]),
    "mpig_lsh_collision_counts": (_i, [_vp, _i, _vp, _vp, _vp]),
    "mpig_lsh_table_ptrs": (_i, [_vp, _i, ctypes.POINTER(_vp), ctypes.POINTER(_vp)]),
    "mpig_attn_fill": (_i, [_vp, _i, _i, _vp, _vp, _vp, _i, _vp]),
    "mpig_attention_wrapper": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mpig_attn_read_cache": (_i, [_vp, _i, _vp, _vp, _vp, _vp]),
    "mpig_simhash": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "mpig_window_fill": (_i, [_vp, _i, _i, _vp, _vp, _vp, _i, _vp]),
    "mpig_plan": (_i, [_vp, _vp]),
    "mpig_spill_window": (_i, [_vp, _i, ctypes.POINTER(ctypes.c_int32), _vp]),
    "mpig_compact_context": (_i, [_vp, _i, ctypes.POINTER(ctypes.c_int32), _vp]),
    "mpig_read_visibility": (_i, [_vp, _vp, _vp]),
    "mpig_decode": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "mpig_decode_timed": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "mpig_timing_collect": (_i, [_vp, ctypes.POINTER(ctypes.c_float), _i, ctypes.POINTER(_i)]),
    "mpig_decode_host": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "mpig_last_probe": (_i, [_vp, _vp, _vp, _vp]),
    "mpig_dense_fill": (_i, [_vp, _i, _i, _vp, _vp, _i, _vp]),
    "mpig_dense_decode": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "mpig_reserve_query_tokens": (_i, [_vp, _i]),
    "mpig_plan_tokens": (_i, [_vp, _i, _vp]),
    "mpig_decode_tokens": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "mpig_dense_decode_tokens": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "mpig_rewind": (_i, [_vp, _vp, _vp]),
    "mpig_plan_tree": (_i, [_vp, _i, _vp, _vp]),
    "mpig_accept": (_i, [_vp, _vp, _vp, _vp]),
    "mpig_reserve_chunk_tokens": (_i, [_vp, _i]),
    "mpig_plan_chunk": (_i, [_vp, _i, _vp]),
    "mpig_chunk_attend": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "mpig_prefill_attend": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "mpig_fork_request": (_i, [_vp, _i, _i, _vp]),
    "mpig_bind_request": (_i, [_vp, _i, _i, _vp]),
    "mpig_reorder_requests": (_i, [_vp, _vp, _vp]),
    "mpig_launch_count": (ctypes.c_uint64, [_vp]),
    "mpig_get_info": (_i, [_vp, ctypes.c_char_p, ctypes.POINTER(ctypes.c_int64)]),
    "mpig_error_flags": (_i, [_vp, ctypes.POINTER(ctypes.c_int32), _vp]),
    "mpig_last_out_f32": (_i, [_vp, _vp, _vp]),
    "mpig_last_codes": (_i, [_vp, _vp, _vp]),
    "mpig_peer_create": (_i, [_vp, _i, _i, ctypes.c_size_t, ctypes.POINTER(_vp)]),
    "mpig_peer_handle": (_i, [_vp, _vp]),
    "mpig_peer_connect": (_i, [_vp, _vp]),
    "mpig_peer_destroy": (None, [_vp]),
    "mpig_peer_all_gather": (_i, [_vp, _vp, _vp, ctypes.c_size_t, _vp]),
    "mpig_peer_all_reduce_bf16": (_i, [_vp, _vp, ctypes.c_size_t, _vp]),
    "mpig_decode_allgather": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mpig_peer_wait_gather": (_i, [_vp, _vp, ctypes.c_size_t, _i, _vp]),
    "mpig_peer_timeouts": (_i, [_vp, ctypes.POINTER(ctypes.c_ulonglong)]),
    "mpig_debug_read": (_i, [_vp, _vp, _i]),
    "mpig_fused_debug_read": (_i, [_vp, _vp, _i]),
}


# harness-side helpers declared in include/magicpig_b200_aux.h (not part of the drop-in boundary)
_AUX_SIGNATURES = {
    "mpig_aux_add_rmsnorm": (_i, [_vp, _vp, _vp, ctypes.c_float, _vp, _i, _i, _vp]),
    "mpig_aux_rope_split": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "mpig_aux_silu_mul": (_i, [_vp, _vp, _i, _i, _vp]),
    "mpig_aux_gemv": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "mpig_aux_norm_gemv": (_i, [_vp, _vp, _vp, _vp, ctypes.c_float, _vp, _vp, _i, _i, _i, _i, _vp]),
    "mpig_aux_set_pdl": (_i, [_i]),
    "mpig_aux_norm_qkv_rope": (_i, [_vp, _vp, _vp, _vp, ctypes.c_float, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "mpig_aux_sample": (_i, [_vp, _i, _i, ctypes.c_int64, _vp, _vp, ctypes.c_uint64, _vp, _vp, ctypes.c_int64, _vp, _vp, _vp, _i,
                             _vp, _i, _vp, _vp, _vp, _vp]),
    "mpig_aux_sample_occupancy": (_i, [_i, ctypes.POINTER(_i)]),
    "mpig_aux_verify_sample": (_i, [_vp, _i, _i, _i, ctypes.c_int64, ctypes.c_int64, _vp, _vp, ctypes.c_uint64, _vp, _vp,
                                    ctypes.c_int64, _vp, _vp, _vp, ctypes.c_int64, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp,
                                    _vp]),
    "mpig_aux_sample_filtered": (_i, [_vp, _i, _i, ctypes.c_int64, _vp, _vp, ctypes.c_uint64, _vp, _vp, ctypes.c_int64, _vp, _vp, _vp,
                                      _i, _vp, _i, _vp, _vp, _vp, ctypes.POINTER(MpigSampleFilters), _vp]),
    "mpig_aux_verify_sample_filtered": (_i, [_vp, _i, _i, _i, ctypes.c_int64, ctypes.c_int64, _vp, _vp, ctypes.c_uint64, _vp, _vp,
                                             ctypes.c_int64, _vp, _vp, _vp, ctypes.c_int64, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp,
                                             _vp, ctypes.POINTER(MpigSampleFilters), _vp]),
    "mpig_aux_ngram_draft": (_i, [_vp, _i, ctypes.c_int64, _vp, _vp, ctypes.c_int64, _i, _i, _i, _vp]),
}


AUX_HEADER_PATH = os.path.join(_HERE, "..", "include", "magicpig_b200_aux.h")


def declared_symbols(header: str = HEADER_PATH) -> list[str]:
    """Every entry point a header under include/ declares (parsed from the header text)."""
    with open(header) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(mpig_[a-z0-9_]+)\s*\(", text)))


def load() -> ctypes.CDLL:
    """Load the CUDA library.  Fails loudly when it has not been built (no fallback exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MagicPigError(
            f"{LIB_PATH} is missing: build it with `python -m magicpig_b200.build` "
            "(or __graft_entry__.build()).  magicpig_b200 has no CPU/PyTorch fallback.")
    import torch  # noqa: F401  -- loads libcudart.so.12 first so both sides share one CUDA runtime

    lib = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    for name, (res, args) in list(_SIGNATURES.items()) + list(_AUX_SIGNATURES.items()):
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if lib.mpig_abi_version() != MPIG_ABI_VERSION:
        raise MagicPigError(f"ABI mismatch: library {lib.mpig_abi_version()} vs binding {MPIG_ABI_VERSION}")
    _lib = lib
    return lib


def check(rc: int, what: str = ""):
    if rc != MPIG_OK:
        msg = load().mpig_last_error().decode(errors="replace")
        raise MagicPigError(f"{what or 'magicpig_b200'} failed (code {rc}): {msg}")
