"""Host-side mirror of the reference's native operator surface, on top of the C ABI.

`Context` is a thin torch-tensor front-end of `mpig_ctx` (include/magicpig_b200.h).  `LSH` and
`SparseAttentionServer` keep the NAMES, argument order and in-place output convention of the two
reference pybind classes so that parity tests read like the reference's own tests:

    lsh.LSH                                     library/lsh/lsh.cc:316-326
    sparse_attention_cpu.SparseAttentionServer  library/sparse_attention/sparse_attention.cc:1243-1263

with one difference: tensors live on the GPU (that is the point), and shape/dtype errors raise
instead of being undefined behaviour.  Nothing here computes on the CPU and nothing falls back.
"""
from __future__ import annotations

import ctypes
import math
import os
from dataclasses import dataclass
from typing import Optional, Sequence

import torch

from . import _native as N


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream() -> ctypes.c_void_p:
    """The current CUDA stream of the current device as a handle (no Stream object when torch exposes the raw getter)."""
    if _raw_stream is not None:
        return ctypes.c_void_p(_raw_stream(torch.cuda.current_device()))
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


class Context:
    """Owns the HBM-resident KV store, hash tables, window cache and scratch of one model replica/rank."""

    def __init__(self, K: int, L: int, num_layers: int, num_attention_heads: int, num_key_value_heads: int,
                 head_dim: int, batch_size: int, max_length: int, num_sink_tokens: int = 4, num_local_tokens: int = 64,
                 generation_buffer: int = 256, dense_layers: Sequence[int] = (), alloc_dense_kv: bool = False,
                 device: str | torch.device = "cuda:0", max_query_tokens: int = 1, num_contexts: int = 0,
                 dense_tail_rows: int = 0, shared_spill: bool = False):
        """num_contexts: context slots C in [0, batch_size] (0 = batch_size, every request owns its context).  The sampled store
        and the hash tables exist once per slot; requests bound to one slot decode over one copy (fork(), bind()).
        dense_tail_rows: R > 0 keeps the dense layers' prompt rows once per slot as well (needs C < batch_size and alloc_dense_kv);
        each request holds only the R rows it adds after its prompt, so it may generate at most R tokens past the prompt it was
        filled or forked with.  0 = one full dense cache per request.
        shared_spill: requests that share a slot may spill_window() into it (needs 0 < C < batch_size <= 32).  Each spilled key is
        private: it is seen by the request that spilled it and by requests later forked from it, so every request decodes as if
        it had the slot to itself.  Private keys nobody sees any more keep their place in the slot until it is refilled or
        compact() reclaims them: size max_length for the prompt plus the spilled tokens still seen and one spill."""
        self.lib = N.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise N.MagicPigError("magicpig_b200 runs on CUDA (sm_90a) only; there is no CPU path")
        self.K, self.L, self.num_layers = K, L, num_layers
        self.Hq, self.Hkv, self.d = num_attention_heads, num_key_value_heads, head_dim
        self.B, self.M = batch_size, max_length
        self.H = self.B * self.Hq
        self.G = self.Hq // max(self.Hkv, 1)
        self.NB = 1 << K
        self.num_sink_tokens, self.num_local_tokens = num_sink_tokens, num_local_tokens
        self.Wcap = num_sink_tokens + num_local_tokens + generation_buffer
        self.dense_layers = sorted(set(int(x) for x in dense_layers if 0 <= int(x) < num_layers))
        cfg = N.MpigConfig()
        cfg.abi_version = N.MPIG_ABI_VERSION
        cfg.device = self.device.index or 0
        cfg.K, cfg.L, cfg.num_layers = K, L, num_layers
        cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim = num_attention_heads, num_key_value_heads, head_dim
        cfg.batch_size, cfg.max_length = batch_size, max_length
        cfg.num_sink_tokens, cfg.num_local_tokens, cfg.generation_buffer = num_sink_tokens, num_local_tokens, generation_buffer
        if len(self.dense_layers) > 16:
            raise N.MagicPigError("at most 16 dense layers")
        cfg.num_dense_layers = len(self.dense_layers)
        for i, l in enumerate(self.dense_layers):
            cfg.dense_layers[i] = l
        cfg.alloc_dense_kv = 1 if alloc_dense_kv else 0
        cfg.ctas_per_sm = int(os.environ.get("MPIG_CTA_PER_SM", "1"))   # experiment switch: 2 = clusters of 512-thread CTAs, two per SM
        cfg.num_contexts = int(num_contexts)
        cfg.dense_tail_rows = int(dense_tail_rows)
        cfg.shared_spill = 1 if shared_spill else 0
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            N.check(self.lib.mpig_create(ctypes.byref(cfg), ctypes.byref(h)), "mpig_create")
        self._h = h
        self.C = self.get_info("num_contexts")
        self.dense_tail_rows = self.get_info("dense_tail_rows")
        self.shared_spill = bool(self.get_info("shared_spill"))
        self.max_query_tokens = 1
        self.last_tokens = 1   # T of the last decode: the readers return B*T*Hq rows
        self.pending_tokens = 0   # T of the last plan (the shape accept() expects)
        self.pending_chunk = False   # the last plan was plan_chunk(): the layers' calls of the step are chunk_attend()
        self.max_chunk_tokens = 0
        if max_query_tokens > 1:
            self.reserve_query_tokens(max_query_tokens)

    # -- lifetime ---------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            self.lib.mpig_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def device_bytes(self) -> int:
        return int(self.lib.mpig_device_bytes(self._h))

    @property
    def launch_count(self) -> int:
        return int(self.lib.mpig_launch_count(self._h))

    def set_option(self, key: str, value: int):
        N.check(self.lib.mpig_set_option(self._h, key.encode(), int(value)), "mpig_set_option")

    def clear(self):
        N.check(self.lib.mpig_clear(self._h, _stream()), "mpig_clear")
        self.last_tokens = 1
        self.pending_tokens = 0
        self.pending_chunk = False

    @property
    def num_contexts(self) -> int:
        return self.C

    def fork(self, src: int, dst: int):
        """Bind request dst to request src's context slot and copy src's window, avg_k, dense-layer KV and lengths into dst
        (with dense_tail_rows > 0 only the dense rows past src's prompt: the prompt stays in the slot).  With shared_spill dst
        sees exactly the spilled keys src sees.
        Synchronises; not capturable, but a step captured before it replays with the new binding.  Ends the pending step
        (rewind / accept are refused until the next plan)."""
        N.check(self.lib.mpig_fork_request(self._h, int(src), int(dst), _stream()), "mpig_fork_request")
        self.pending_tokens = 0

    def bind(self, request: int, slot: int):
        """Bind `request` to context slot `slot` without touching its window or lengths (fill the slot and the window next; with
        dense_tail_rows > 0 dense-fill it too before its dense outputs mean anything).  With shared_spill it sees no spilled key
        until it spills again.
        Synchronises; ends the pending step like fork()."""
        N.check(self.lib.mpig_bind_request(self._h, int(request), int(slot), _stream()), "mpig_bind_request")
        self.pending_tokens = 0

    def reorder(self, src_of: torch.Tensor):
        """Request b continues request src_of[b]'s sequence: fork(src_of[b], b) for every b with src_of[b] != b, in one kernel
        on the device.  src_of: int32 (B,) on the device; every source must keep its own sequence (src_of[src_of[b]] ==
        src_of[b]).  Capturable: a replay reorders by whatever src_of holds then.  Eager calls synchronise and raise on a map that
        breaks the rule without changing anything; under capture such a map changes nothing and raises error_flags() bit 4.
        Ends the pending step like fork()."""
        self._chk(src_of, torch.int32, (self.B,), "src_of")
        N.check(self.lib.mpig_reorder_requests(self._h, _ptr(src_of), _stream()), "mpig_reorder_requests")
        self.pending_tokens = 0

    def get_info(self, key: str) -> int:
        v = ctypes.c_int64(0)
        N.check(self.lib.mpig_get_info(self._h, key.encode(), ctypes.byref(v)), "mpig_get_info")
        return int(v.value)

    def error_flags(self) -> int:
        """bit 0: a sparse window is full (generation_buffer exhausted), bit 1: a dense cache reached its capacity, bit 2: a rewind drop was out
        of range, bit 3: a malformed tree or accepted path, bit 4: a reorder map that breaks its rule.  Synchronises."""
        f = ctypes.c_int32(0)
        N.check(self.lib.mpig_error_flags(self._h, ctypes.byref(f), _stream()), "mpig_error_flags")
        return int(f.value)

    def last_out_f32(self) -> torch.Tensor:
        """fp32 (B*T*Hq, d) output of the last decode (T = 1 for single-token decodes) before the ABI's bf16 rounding
        (set_option("out_f32", 1) first)."""
        out = torch.empty((self.H * self.last_tokens, self.d), dtype=torch.float32, device=self.device)
        N.check(self.lib.mpig_last_out_f32(self._h, _ptr(out), _stream()), "mpig_last_out_f32")
        return out

    def last_codes(self) -> torch.Tensor:
        """int32 (B*T*Hq, L) query codes the last decode probed with (fused decode: set_option("save_mask", 1) first)."""
        codes = torch.empty((self.H * self.last_tokens, self.L), dtype=torch.int32, device=self.device)
        N.check(self.lib.mpig_last_codes(self._h, _ptr(codes), _stream()), "mpig_last_codes")
        return codes

    def fused_debug_read(self, nctas: int):
        """[[16 clock stamps] per CTA] of the fused kernel's debug instantiation (set_option("fused_debug", 1) first)."""
        buf = (ctypes.c_ulonglong * (16 * nctas))()
        torch.cuda.synchronize(self.device)
        N.check(self.lib.mpig_fused_debug_read(self._h, ctypes.cast(buf, ctypes.c_void_p), nctas), "mpig_fused_debug_read")
        return [[int(buf[16 * i + k]) for k in range(16)] for i in range(nctas)]

    # -- checks -----------------------------------------------------------------------------
    def _chk(self, t: torch.Tensor, dtype, shape, name):
        if t.device != self.device:
            raise N.MagicPigError(f"{name}: expected a tensor on {self.device}, got {t.device}")
        if t.dtype != dtype:
            raise N.MagicPigError(f"{name}: expected dtype {dtype}, got {t.dtype}")
        if shape is not None and tuple(t.shape) != tuple(shape):
            raise N.MagicPigError(f"{name}: expected shape {tuple(shape)}, got {tuple(t.shape)}")
        if not t.is_contiguous():
            raise N.MagicPigError(f"{name}: must be contiguous")
        return t

    # -- hash function ----------------------------------------------------------------------
    def set_hash_func(self, hash_func: torch.Tensor):
        self._chk(hash_func, torch.bfloat16, (self.d, self.K * self.L), "hash_func")
        N.check(self.lib.mpig_set_hash_func(self._h, _ptr(hash_func), _stream()), "mpig_set_hash_func")

    # -- LSH --------------------------------------------------------------------------------
    def lsh_fill(self, layer: int, request: int, sorted_codes: torch.Tensor, sorted_indices: torch.Tensor):
        n = sorted_codes.shape[-1]
        self._chk(sorted_codes, torch.int16, (self.Hkv, self.L, n), "sorted_hash_code")
        self._chk(sorted_indices, torch.int32, (self.Hkv, self.L, n), "sorted_indices")
        N.check(self.lib.mpig_lsh_fill(self._h, layer, request, _ptr(sorted_codes), _ptr(sorted_indices), n, _stream()),
                "mpig_lsh_fill")

    def hash_keys(self, keys: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Key-side SimHash on the tensor cores: keys bf16 (Hkv, n, d) -> codes int16 (Hkv, L, n)."""
        n = keys.shape[1]
        self._chk(keys, torch.bfloat16, (self.Hkv, n, self.d), "keys")
        if out is None:
            out = torch.empty((self.Hkv, self.L, n), dtype=torch.int16, device=self.device)
        else:
            self._chk(out, torch.int16, (self.Hkv, self.L, n), "codes")
        N.check(self.lib.mpig_hash_keys(self._h, _ptr(keys), n, _ptr(out), _stream()), "mpig_hash_keys")
        return out

    def lsh_build(self, layer: int, request: int, key_codes: torch.Tensor):
        n = key_codes.shape[-1]
        self._chk(key_codes, torch.int16, (self.Hkv, self.L, n), "key_codes")
        N.check(self.lib.mpig_lsh_build(self._h, layer, request, _ptr(key_codes), n, _stream()), "mpig_lsh_build")

    def lsh_batch_retrieve(self, layer: int, query: torch.Tensor, results: torch.Tensor, nnz: torch.Tensor):
        self._chk(query, torch.int32, (self.H, self.L), "query")
        self._chk(results, torch.int32, (self.H, self.M), "results")
        self._chk(nnz, torch.int32, (self.H,), "nnz")
        N.check(self.lib.mpig_lsh_batch_retrieve(self._h, layer, _ptr(query), _ptr(results), _ptr(nnz), _stream()),
                "mpig_lsh_batch_retrieve")

    def lsh_get_mask(self) -> torch.Tensor:
        mask = torch.empty((self.B, self.Hq, self.M), dtype=torch.uint8, device=self.device)
        N.check(self.lib.mpig_lsh_get_mask(self._h, _ptr(mask), _stream()), "mpig_lsh_get_mask")
        return mask

    def lsh_collision_counts(self, layer: int, query: torch.Tensor) -> torch.Tensor:
        self._chk(query, torch.int32, (self.H, self.L), "query")
        counts = torch.empty((self.H, self.M), dtype=torch.int32, device=self.device)
        N.check(self.lib.mpig_lsh_collision_counts(self._h, layer, _ptr(query), _ptr(counts), _stream()),
                "mpig_lsh_collision_counts")
        return counts

    # -- KV store + attention -----------------------------------------------------------------
    def attn_fill(self, layer: int, request: int, k: torch.Tensor, v: torch.Tensor, kn: torch.Tensor):
        n = k.shape[1]
        self._chk(k, torch.bfloat16, (self.Hkv, n, self.d), "k")
        self._chk(v, torch.bfloat16, (self.Hkv, n, self.d), "v")
        self._chk(kn, torch.float32, (self.Hkv, n), "kn")
        N.check(self.lib.mpig_attn_fill(self._h, layer, request, _ptr(k), _ptr(v), _ptr(kn), n, _stream()), "mpig_attn_fill")

    def attention_wrapper(self, layer: int, K: int, L: int, output: torch.Tensor, max_value_expsum: torch.Tensor,
                          query: torch.Tensor, query_norm: torch.Tensor, ind: torch.Tensor, nnz: torch.Tensor):
        self._chk(output, torch.bfloat16, (self.H, self.d), "output")
        self._chk(max_value_expsum, torch.float32, (2, self.H), "max_value_expsum")
        if query.dim() != 2:
            query = query.reshape(self.H, self.d)
        self._chk(query, torch.bfloat16, (self.H, self.d), "query")
        query_norm = query_norm.reshape(self.H)
        self._chk(query_norm, torch.float32, (self.H,), "query_norm")
        self._chk(ind, torch.int32, (self.H, self.M), "ind")
        self._chk(nnz, torch.int32, (self.H,), "nnz")
        N.check(self.lib.mpig_attention_wrapper(self._h, layer, K, L, _ptr(output), _ptr(max_value_expsum), _ptr(query),
                                                _ptr(query_norm), _ptr(ind), _ptr(nnz), _stream()), "mpig_attention_wrapper")
        self.last_tokens = 1

    def read_cache(self, layer: int, want_k=True, want_v=True, want_kn=True):
        """k, v (C, Hkv, M, d) bf16 and kn (C, Hkv, M) fp32: the sampled store of every context slot (C = B by default)."""
        k = torch.empty((self.C, self.Hkv, self.M, self.d), dtype=torch.bfloat16, device=self.device) if want_k else None
        v = torch.empty((self.C, self.Hkv, self.M, self.d), dtype=torch.bfloat16, device=self.device) if want_v else None
        kn = torch.empty((self.C, self.Hkv, self.M), dtype=torch.float32, device=self.device) if want_kn else None
        N.check(self.lib.mpig_attn_read_cache(self._h, layer, _ptr(k), _ptr(v), _ptr(kn), _stream()), "mpig_attn_read_cache")
        return k, v, kn

    # -- decode glue ------------------------------------------------------------------------
    def simhash(self, query: torch.Tensor, want_norm: bool = True):
        query = query.reshape(self.H, self.d)
        self._chk(query, torch.bfloat16, (self.H, self.d), "query")
        codes = torch.empty((self.H, self.L), dtype=torch.int32, device=self.device)
        qn = torch.empty((self.H,), dtype=torch.float32, device=self.device) if want_norm else None
        N.check(self.lib.mpig_simhash(self._h, _ptr(query), _ptr(codes), _ptr(qn), _stream()), "mpig_simhash")
        return codes, qn

    def window_fill(self, layer: int, request: int, avg_k: torch.Tensor, k: torch.Tensor, v: torch.Tensor):
        w = k.shape[1]
        self._chk(avg_k, torch.bfloat16, (self.Hkv, self.d), "avg_k")
        self._chk(k, torch.bfloat16, (self.Hkv, w, self.d), "window k")
        self._chk(v, torch.bfloat16, (self.Hkv, w, self.d), "window v")
        N.check(self.lib.mpig_window_fill(self._h, layer, request, _ptr(avg_k), _ptr(k), _ptr(v), w, _stream()),
                "mpig_window_fill")

    def plan(self, tokens: int = 1, parents: Optional[torch.Tensor] = None):
        """Advance every request's lengths by `tokens` (a verification step of that many tokens; reserve them first).  With
        `parents` (device int32 (B, tokens): parents[b][0] = -1, 0 <= parents[b][t] < t) the step is a token tree: node t attends to
        the context, its ancestors and itself.  Capturable; eager calls raise on a malformed tree without changing anything."""
        if parents is not None:
            self._chk(parents, torch.int32, (self.B, int(tokens)), "parents")
            N.check(self.lib.mpig_plan_tree(self._h, int(tokens), _ptr(parents), _stream()), "mpig_plan_tree")
        elif tokens == 1:
            N.check(self.lib.mpig_plan(self._h, _stream()), "mpig_plan")
        else:
            N.check(self.lib.mpig_plan_tokens(self._h, int(tokens), _stream()), "mpig_plan_tokens")
        self.pending_tokens = int(tokens)
        self.pending_chunk = False

    def reserve_chunk_tokens(self, t_max: int):
        """Allocate the scratch of chunk steps of up to t_max <= 1024 tokens (plan_chunk / chunk_attend).  Not capturable, and
        refused once a step has been captured into a CUDA graph: reserve before capturing."""
        N.check(self.lib.mpig_reserve_chunk_tokens(self._h, int(t_max)), "mpig_reserve_chunk_tokens")
        self.max_chunk_tokens = max(self.max_chunk_tokens, int(t_max))

    def plan_chunk(self, T: int):
        """Advance every request's lengths by T for a chunk step: T new prompt tokens per request, which every layer then attends
        with chunk_attend() (exact causal attention over the whole context).  rewind() afterwards makes the chunk ragged.
        Capturable; eager calls raise, changing nothing, when T does not fit a window or a dense cache."""
        N.check(self.lib.mpig_plan_chunk(self._h, int(T), _stream()), "mpig_plan_chunk")
        self.pending_tokens = int(T)
        self.pending_chunk = True

    def chunk_attend(self, layer: int, T: int, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor,
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Sparse or dense layer, chunk step of T tokens: query (B,T,Hq,d), key/value (B,T,Hkv,d) bf16 -> out (B, T, Hq*d).  Token
        t attends exactly (softmax over every key, no sampling) to the request's context and the chunk's tokens up to t."""
        q, k, v, out = self._decode_args(T, query, key, value, out, (self.B, T, self.Hq * self.d))
        N.check(self.lib.mpig_chunk_attend(self._h, layer, int(T), _ptr(q), _ptr(k), _ptr(v), _ptr(out), _stream()),
                "mpig_chunk_attend")
        self.last_tokens = int(T)
        return out

    def prefill_attend(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: Optional[torch.Tensor] = None,
                       out_f32: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Exact causal attention of a prompt chunk over its keys: q (q_len, Hq, d), k / v (kv_len, Hkv, d) bf16 NHD -> out (q_len, Hq, d)
        bf16; query i sees keys [0, kv_len - q_len + i].  out_f32 (q_len, Hq, d) fp32, when given, receives the same values before the
        bf16 rounding.  Uses no context state (any layer, any pending step); capturable."""
        q_len, kv_len = q.shape[0], k.shape[0]
        self._chk(q, torch.bfloat16, (q_len, self.Hq, self.d), "q")
        self._chk(k, torch.bfloat16, (kv_len, self.Hkv, self.d), "k")
        self._chk(v, torch.bfloat16, (kv_len, self.Hkv, self.d), "v")
        if out is None:
            out = torch.empty((q_len, self.Hq, self.d), dtype=torch.bfloat16, device=self.device)
        else:
            self._chk(out, torch.bfloat16, (q_len, self.Hq, self.d), "out")
        if out_f32 is not None:
            self._chk(out_f32, torch.float32, (q_len, self.Hq, self.d), "out_f32")
        N.check(self.lib.mpig_prefill_attend(self._h, _ptr(q), _ptr(k), _ptr(v), int(q_len), int(kv_len), _ptr(out), _ptr(out_f32),
                                             _stream()), "mpig_prefill_attend")
        return out

    def accept(self, nodes: torch.Tensor, count: torch.Tensor):
        """Commit the root path nodes[b][0 .. count[b]) of the pending step of request b: the path's rows move to the front of
        the step in every sparse window and dense cache, and both lengths become base + count[b].  nodes: int32 (B, T), count: int32
        (B,) on the device.  Capturable; eager calls raise on a path that is not a root path of the step without changing anything
        (the call may be repeated)."""
        self._chk(nodes, torch.int32, (self.B, self.pending_tokens), "nodes")
        self._chk(count, torch.int32, (self.B,), "count")
        N.check(self.lib.mpig_accept(self._h, _ptr(nodes), _ptr(count), _stream()), "mpig_accept")

    def reserve_query_tokens(self, t_max: int):
        """Allocate the per-step scratch for verification steps of up to t_max <= 8 tokens.  Not capturable, and refused once a
        step has been captured into a CUDA graph (the scratch moves): reserve before capturing."""
        N.check(self.lib.mpig_reserve_query_tokens(self._h, int(t_max)), "mpig_reserve_query_tokens")
        self.max_query_tokens = max(self.max_query_tokens, int(t_max))

    def rewind(self, drop: torch.Tensor):
        """Drop the last drop[b] tokens of the pending step of request b; drop: int32 (B,) on the device.  Capturable; eager
        calls synchronise and raise on a drop outside [0, T] without changing anything (the call may be repeated)."""
        self._chk(drop, torch.int32, (self.B,), "drop")
        N.check(self.lib.mpig_rewind(self._h, _ptr(drop), _stream()), "mpig_rewind")

    def _decode_args(self, T: int, query, key, value, out, out_shape):
        """The rows of a step of T tokens per request (T = 1: a single-token decode): query / key / value flattened to
        (B*T*Hq, d) / (B*T*Hkv, d) and checked, and `out` checked, or allocated with out_shape when None."""
        q = query.reshape(self.B * T * self.Hq, self.d)
        k = key.reshape(self.B * T * self.Hkv, self.d)
        v = value.reshape(self.B * T * self.Hkv, self.d)
        self._chk(q, torch.bfloat16, None, "query")
        self._chk(k, torch.bfloat16, None, "key")
        self._chk(v, torch.bfloat16, None, "value")
        if out is None:
            out = torch.empty(out_shape, dtype=torch.bfloat16, device=self.device)
        else:
            self._chk(out, torch.bfloat16, None, "out")
            if out.numel() != self.B * T * self.Hq * self.d:
                raise N.MagicPigError(f"out: expected {self.B * T * self.Hq * self.d} elements, got {out.numel()}")
        return q, k, v, out

    def decode_tokens(self, layer: int, T: int, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor,
                      out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Sparse layer, verification step of T tokens: query (B,T,Hq,d), key/value (B,T,Hkv,d) bf16 -> out (B, T, Hq*d)."""
        q, k, v, out = self._decode_args(T, query, key, value, out, (self.B, T, self.Hq * self.d))
        N.check(self.lib.mpig_decode_tokens(self._h, layer, int(T), _ptr(q), _ptr(k), _ptr(v), _ptr(out), _stream()),
                "mpig_decode_tokens")
        self.last_tokens = int(T)
        return out

    def dense_decode_tokens(self, layer: int, T: int, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor,
                            out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Dense layer, same shapes as decode_tokens."""
        q, k, v, out = self._decode_args(T, query, key, value, out, (self.B, T, self.Hq * self.d))
        N.check(self.lib.mpig_dense_decode_tokens(self._h, layer, int(T), _ptr(q), _ptr(k), _ptr(v), _ptr(out), _stream()),
                "mpig_dense_decode_tokens")
        self.last_tokens = int(T)
        return out

    def spill_window(self, keep: Optional[int] = None) -> torch.Tensor:
        """Move the oldest non-sink window rows of every request and sparse layer into the sampled store and the hash tables,
        keeping the newest `keep` (default num_local_tokens) in the window.  Returns the spilled row count per request, int32 (B,)
        on the host.  Synchronises; not capturable, but a decode step captured before the spill stays valid after it."""
        keep = self.num_local_tokens if keep is None else int(keep)
        out = (ctypes.c_int32 * self.B)()
        N.check(self.lib.mpig_spill_window(self._h, keep, out, _stream()), "mpig_spill_window")
        return torch.tensor(list(out), dtype=torch.int32)

    def compact(self, slot: Optional[int] = None) -> torch.Tensor:
        """shared_spill only: drop the spilled keys that no request sees any more (their owner was forked over, reordered over,
        rebound or retired) from the store and the tables of context slot `slot` (None: every slot), in place.  Every request
        samples exactly what it sampled before; the live keys keep their time order at the lowest offsets.  Returns the keys
        reclaimed per slot, int32 (C,) on the host (zeros without shared_spill).  Synchronises; not capturable, but a decode step
        captured before the call stays valid after it."""
        out = (ctypes.c_int32 * self.C)()
        N.check(self.lib.mpig_compact_context(self._h, -1 if slot is None else int(slot), out, _stream()), "mpig_compact_context")
        return torch.tensor(list(out), dtype=torch.int32)

    def visibility(self) -> torch.Tensor:
        """Diagnostic accessor, shared_spill only: a copy of the visibility map, int32 (C, max_length) on the device; bit b of
        [c, p] = request b sees the spilled key at private offset p of slot c."""
        out = torch.empty((self.C, self.M), dtype=torch.int32, device=self.device)
        N.check(self.lib.mpig_read_visibility(self._h, _ptr(out), _stream()), "mpig_read_visibility")
        return out

    def decode(self, layer: int, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor,
               out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """query (B,Hq,1,d)|(B*Hq,d), key/value (B,Hkv,1,d)|(B*Hkv,d) bf16 -> out (B, Hq*d) bf16."""
        q, k, v, out = self._decode_args(1, query, key, value, out, (self.B, self.Hq * self.d))
        N.check(self.lib.mpig_decode(self._h, layer, _ptr(q), _ptr(k), _ptr(v), _ptr(out), _stream()), "mpig_decode")
        self.last_tokens = 1
        return out

    def decode_timed(self, layer: int, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, out: torch.Tensor):
        """decode() with CUDA events between the three kernels.  Asynchronous: read the times of all calls since the
        last collect with timing_collect()."""
        q, k, v, out = self._decode_args(1, query, key, value, out, (self.B, self.Hq * self.d))
        N.check(self.lib.mpig_decode_timed(self._h, layer, _ptr(q), _ptr(k), _ptr(v), _ptr(out), _stream()), "mpig_decode_timed")
        self.last_tokens = 1

    def timing_collect(self, max_calls: int = 4096):
        """[(simhash_ms, probe_ms, attend_ms), ...] for every decode_timed() since the last collect (synchronises)."""
        buf = (ctypes.c_float * (3 * max_calls))()
        n = ctypes.c_int(0)
        N.check(self.lib.mpig_timing_collect(self._h, buf, max_calls, ctypes.byref(n)), "mpig_timing_collect")
        return [(buf[3 * i], buf[3 * i + 1], buf[3 * i + 2]) for i in range(n.value)]

    def decode_host(self, layer: int, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, out: torch.Tensor):
        """Same with HOST (pinned) tensors; synchronous like the reference's CPU operators."""
        bf16 = torch.bfloat16
        if not (query.is_cpu and key.is_cpu and value.is_cpu and out.is_cpu and query.dtype is bf16 and key.dtype is bf16
                and value.dtype is bf16 and out.dtype is bf16 and query.is_contiguous() and key.is_contiguous()
                and value.is_contiguous() and out.is_contiguous()):
            raise N.MagicPigError("decode_host: query / key / value / out must be contiguous CPU bf16 tensors")
        nq, nk = self.H * self.d, self.B * self.Hkv * self.d
        if query.numel() != nq or out.numel() != nq or key.numel() != nk or value.numel() != nk:
            raise N.MagicPigError(f"decode_host: expected {nq} query/out and {nk} key/value elements")
        rc = self.lib.mpig_decode_host(self._h, layer, query.data_ptr(), key.data_ptr(), value.data_ptr(), out.data_ptr(), _stream())
        if rc:
            N.check(rc, "mpig_decode_host")
        self.last_tokens = 1
        return out

    def last_probe(self, want_results: bool = False):
        """nnz (B*T*Hq,) int32 [and results (B*T*Hq, M)] of the most recent decode's probe (T = 1 for single-token decodes)."""
        rows = self.H * self.last_tokens
        nnz = torch.empty((rows,), dtype=torch.int32, device=self.device)
        res = torch.empty((rows, self.M), dtype=torch.int32, device=self.device) if want_results else None
        N.check(self.lib.mpig_last_probe(self._h, _ptr(nnz), _ptr(res), _stream()), "mpig_last_probe")
        return nnz, res

    # -- dense layers -----------------------------------------------------------------------
    def dense_fill(self, layer: int, request: int, k: torch.Tensor, v: torch.Tensor, seq_len: int):
        self._chk(k, torch.bfloat16, None, "k")
        self._chk(v, torch.bfloat16, None, "v")
        if k.shape[0] < seq_len or tuple(k.shape[1:]) != (self.Hkv, self.d):
            raise N.MagicPigError(f"dense_fill: k must be (>= {seq_len}, {self.Hkv}, {self.d}), got {tuple(k.shape)}")
        N.check(self.lib.mpig_dense_fill(self._h, layer, request, _ptr(k), _ptr(v), seq_len, _stream()), "mpig_dense_fill")

    def dense_decode(self, layer: int, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor,
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
        q, k, v, out = self._decode_args(1, query, key, value, out, (self.B, self.Hq * self.d))
        N.check(self.lib.mpig_dense_decode(self._h, layer, _ptr(q), _ptr(k), _ptr(v), _ptr(out), _stream()),
                "mpig_dense_decode")
        self.last_tokens = 1
        return out


MAX_EOS_IDS = 8


def _sample_chk(t, dtype, shape, name, device):
    if not isinstance(t, torch.Tensor):
        raise N.MagicPigError(f"{name}: expected a tensor, got {type(t).__name__}")
    if t.device != device:
        raise N.MagicPigError(f"{name}: expected a tensor on {device}, got {t.device}")
    if t.dtype != dtype:
        raise N.MagicPigError(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise N.MagicPigError(f"{name}: expected shape {tuple(shape)}, got {tuple(t.shape)}")
    return t


def check_sample_args(logits, temperature, top_p, offset, ids_out=None, tokens_out=None, count=None, done=None, eos_token_ids=(),
                      status=None, debug=None, debug_w=None, *, n_debug: int = 5):
    """The argument checks of sample() on any device (no library call): returns (ids_out, max_new, eos ids), ids_out allocated
    when None.  Raises MagicPigError."""
    if not isinstance(logits, torch.Tensor) or logits.dim() != 2:
        raise N.MagicPigError("logits: expected a (B, V) tensor")
    dev = logits.device
    _sample_chk(logits, torch.float32, None, "logits", dev)
    B, V = logits.shape
    if B < 1 or V < 1:
        raise N.MagicPigError(f"logits: empty shape {tuple(logits.shape)}")
    if logits.stride(1) != 1 or logits.stride(0) < V:
        raise N.MagicPigError(f"logits: rows must be contiguous with a stride >= V, got strides {logits.stride()}")
    _sample_chk(temperature, torch.float32, (B,), "temperature", dev)
    _sample_chk(top_p, torch.float32, (B,), "top_p", dev)
    if not isinstance(offset, torch.Tensor) or offset.dtype not in (torch.int64, torch.uint64) or offset.numel() != 1:
        raise N.MagicPigError("offset: expected a one-element int64 / uint64 tensor")
    _sample_chk(offset, offset.dtype, None, "offset", dev)
    for name, t in (("temperature", temperature), ("top_p", top_p)):
        if not t.is_contiguous():
            raise N.MagicPigError(f"{name}: must be contiguous")
    eos = [int(e) for e in eos_token_ids]
    if len(eos) > MAX_EOS_IDS:
        raise N.MagicPigError(f"at most {MAX_EOS_IDS} EOS ids, got {len(eos)}")
    if ids_out is None:
        ids_out = torch.empty((B,), dtype=torch.int64, device=dev)
    _sample_chk(ids_out, torch.int64, None, "ids_out", dev)
    if ids_out.shape[0] != B or ids_out.dim() not in (1, 2):
        raise N.MagicPigError(f"ids_out: expected (B={B},) or (B, n), got {tuple(ids_out.shape)}")
    max_new = 0
    if tokens_out is not None:
        if count is None or done is None:
            raise N.MagicPigError("tokens_out needs count and done")
        _sample_chk(tokens_out, torch.int32, None, "tokens_out", dev)
        if tokens_out.dim() != 2 or tokens_out.shape[0] != B or tokens_out.shape[1] < 1 or not tokens_out.is_contiguous():
            raise N.MagicPigError(f"tokens_out: expected a contiguous (B={B}, max_new >= 1) tensor, got {tuple(tokens_out.shape)}")
        max_new = tokens_out.shape[1]
    elif count is not None or done is not None:
        raise N.MagicPigError("count and done go with tokens_out")
    for name, t, dt, shp in (("count", count, torch.int32, (B,)), ("done", done, torch.int32, (B,)),
                             ("status", status, torch.int32, ((B + 31) // 32,)), ("debug", debug, torch.int64, (B, n_debug)),
                             ("debug_w", debug_w, torch.float32, (B, V))):
        if t is not None:
            _sample_chk(t, dt, shp, name, dev)
            if not t.is_contiguous():
                raise N.MagicPigError(f"{name}: must be contiguous")
    return ids_out, max_new, eos


def sample(logits: torch.Tensor, temperature: torch.Tensor, top_p: torch.Tensor, seed: int, offset: torch.Tensor,
           ids_out: Optional[torch.Tensor] = None, tokens_out: Optional[torch.Tensor] = None, count: Optional[torch.Tensor] = None,
           done: Optional[torch.Tensor] = None, eos_token_ids: Sequence[int] = (), status: Optional[torch.Tensor] = None,
           debug: Optional[torch.Tensor] = None, debug_w: Optional[torch.Tensor] = None, *,
           filters: Optional["SampleFilters"] = None) -> torch.Tensor:
    """One token per row of logits (B, V) fp32 (rows may be strided; elements contiguous) by temperature / top-p sampling on the
    device (mpig_aux_sample, include/magicpig_b200_aux.h, states the exact rule): temperature (B,) fp32 (<= 0: greedy, the first
    argmax), top_p (B,) fp32, offset a device uint64 (1,) tensor (int64 storage is accepted) read as the Philox counter and never
    written.  ids_out: int64 tensor whose elements ids_out[b, 0] (or ids_out[b]) receive the tokens; None = a new int64 (B,)
    tensor.  tokens_out int32 (B, max_new) with count / done int32 (B,): append the token unless done, done on an id in
    eos_token_ids (at most 8) or when count reaches max_new.  status int32 ((B + 31) // 32,): bit b % 32 of word b // 32 is set
    for a row with a NaN or +inf logit or none finite (its token is 0).  debug int64 (B, 5) / debug_w fp32 (B, V): the kernel's
    integer stages and weights.  Every argument is checked here before the call; capturable.  Returns the tensor holding the
    tokens (ids_out).
    filters (keyword only): a SampleFilters adds top-k, min-p and the repetition / presence / frequency penalties
    (mpig_aux_sample_filtered); debug is then (B, 8) and each appended token is counted in filters.table.  None is the call
    above, unchanged."""
    ids_out, max_new, eos = check_sample_args(logits, temperature, top_p, offset, ids_out, tokens_out, count, done, eos_token_ids,
                                              status, debug, debug_w, n_debug=5 if filters is None else 8)
    B, V = logits.shape
    if filters is not None:
        check_filters(filters, B, V, logits.device)
    if logits.device.type != "cuda":
        raise N.MagicPigError("sample runs on CUDA (sm_90a) only; there is no CPU path")
    dev = logits.device
    eos_arr = (ctypes.c_int32 * max(len(eos), 1))(*eos)
    lib = N.load()
    args = (_ptr(logits), B, V, logits.stride(0), _ptr(temperature), _ptr(top_p), ctypes.c_uint64(int(seed) & (2 ** 64 - 1)),
            _ptr(offset), _ptr(ids_out), ids_out.stride(0), _ptr(tokens_out), _ptr(count), _ptr(done), max_new, eos_arr, len(eos),
            _ptr(status), _ptr(debug), _ptr(debug_w))
    with torch.cuda.device(dev):
        if filters is None:
            N.check(lib.mpig_aux_sample(*args, _stream()), "mpig_aux_sample")
        else:
            f = filters.native()
            N.check(lib.mpig_aux_sample_filtered(*args, ctypes.byref(f), _stream()), "mpig_aux_sample_filtered")
    return ids_out


MAX_VERIFY_TOKENS = 8   # rows per request of verify_sample and ngram_draft's T
MAX_NGRAM = 8           # longest suffix ngram_draft matches


def _ids_chk(ids, B, T, dev):
    _sample_chk(ids, torch.int64, None, "ids", dev)
    if ids.dim() != 2 or ids.shape[0] != B or ids.shape[1] < T or ids.stride(1) != 1:
        raise N.MagicPigError(f"ids: expected int64 (B={B}, >= T={T}) with contiguous rows, got {tuple(ids.shape)} strides {ids.stride()}")


def check_verify_args(logits, temperature, top_p, offset, ids, rows=None, drop=None, history=None, length=None, limit=None, done=None,
                      steps=None, accepted=None, eos_token_ids=(), status=None, debug=None, debug_w=None, *, n_debug: int = 9):
    """The argument checks of verify_sample() on any device (no library call): returns (rows, eos ids), rows allocated when None.
    Raises MagicPigError."""
    if not isinstance(logits, torch.Tensor) or logits.dim() != 3:
        raise N.MagicPigError("logits: expected a (B, T, V) tensor")
    B, T, V = logits.shape
    if not 1 <= T <= MAX_VERIFY_TOKENS:
        raise N.MagicPigError(f"logits: T={T} outside [1, {MAX_VERIFY_TOKENS}]")
    if V >= 1 and (logits.stride(2) != 1 or logits.stride(1) < V or logits.stride(0) < (T - 1) * logits.stride(1) + V):
        raise N.MagicPigError(f"logits: rows must be contiguous and must not overlap, got strides {logits.stride()}")
    # the per-request checks are sample()'s, on row 0 of every request
    _, _, eos = check_sample_args(logits[:, 0], temperature, top_p, offset, eos_token_ids=eos_token_ids, status=status)
    dev = logits.device
    _ids_chk(ids, B, T, dev)
    if rows is None:
        rows = torch.empty((B, T, 2), dtype=torch.int32, device=dev)
    if history is not None:
        if length is None or limit is None or done is None:
            raise N.MagicPigError("history needs length, limit and done")
        _sample_chk(history, torch.int32, None, "history", dev)
        if history.dim() != 2 or history.shape[0] != B or history.shape[1] < 1 or not history.is_contiguous():
            raise N.MagicPigError(f"history: expected a contiguous (B={B}, n >= 1) tensor, got {tuple(history.shape)}")
    elif length is not None or limit is not None or done is not None:
        raise N.MagicPigError("length, limit and done go with history")
    if (steps is None) != (accepted is None):
        raise N.MagicPigError("steps and accepted go together")
    for name, t, dt, shp in (("rows", rows, torch.int32, (B, T, 2)), ("drop", drop, torch.int32, (B,)),
                             ("length", length, torch.int32, (B,)), ("limit", limit, torch.int32, (B,)),
                             ("done", done, torch.int32, (B,)), ("steps", steps, torch.int32, (B,)),
                             ("accepted", accepted, torch.int32, (B,)), ("debug", debug, torch.int64, (B, T, n_debug)),
                             ("debug_w", debug_w, torch.float32, (B, T, V))):
        if t is not None:
            _sample_chk(t, dt, shp, name, dev)
            if not t.is_contiguous():
                raise N.MagicPigError(f"{name}: must be contiguous")
    return rows, eos


def verify_sample(logits: torch.Tensor, temperature: torch.Tensor, top_p: torch.Tensor, seed: int, offset: torch.Tensor,
                  ids: torch.Tensor, rows: Optional[torch.Tensor] = None, drop: Optional[torch.Tensor] = None,
                  history: Optional[torch.Tensor] = None, length: Optional[torch.Tensor] = None, limit: Optional[torch.Tensor] = None,
                  done: Optional[torch.Tensor] = None, steps: Optional[torch.Tensor] = None, accepted: Optional[torch.Tensor] = None,
                  eos_token_ids: Sequence[int] = (), status: Optional[torch.Tensor] = None, debug: Optional[torch.Tensor] = None,
                  debug_w: Optional[torch.Tensor] = None, *, filters: Optional["SampleFilters"] = None) -> torch.Tensor:
    """Speculative sampling of a verification step on the device (mpig_aux_verify_sample, include/magicpig_b200_aux.h, states the
    exact rule): logits (B, T, V) fp32 (the logits after each of the step's T inputs; rows may be strided, elements contiguous),
    ids (B, >= T) int64 the step's inputs, so ids[b, 1:T] are request b's drafts.  Accepts a prefix of the drafts and draws the
    final token, which goes to ids[b, 0].  temperature / top_p / seed / offset / status / eos_token_ids as in sample().  rows: int32
    (B, T, 2) scratch (None = allocated).  drop int32 (B,): T - 1 - accepted drafts, the rewind() input.  history int32 (B, n) with
    length / limit / done int32 (B,): the emitted tokens are appended at length[b] until an EOS id or limit[b] sets done[b]; a
    request already done appends nothing and gets drop = T.  steps / accepted int32 (B,): += 1 and += accepted drafts per call.
    debug int64 (B, T, 9) / debug_w fp32 (B, T, V): each row's integer stages and weights.  Every argument is checked here before the
    call; capturable.  Returns ids.
    filters (keyword only): a SampleFilters adds top-k, min-p and the penalties (mpig_aux_verify_sample_filtered): row t also counts
    the drafts ids[b, 1 .. t] in the penalties, debug is (B, T, 12) and each token appended to history is counted in
    filters.table.  None is the call above, unchanged."""
    rows, eos = check_verify_args(logits, temperature, top_p, offset, ids, rows, drop, history, length, limit, done, steps, accepted,
                                  eos_token_ids, status, debug, debug_w, n_debug=9 if filters is None else 12)
    B, T, V = logits.shape
    if filters is not None:
        check_filters(filters, B, V, logits.device)
    if logits.device.type != "cuda":
        raise N.MagicPigError("verify_sample runs on CUDA (sm_90a) only; there is no CPU path")
    eos_arr = (ctypes.c_int32 * max(len(eos), 1))(*eos)
    lib = N.load()
    args = (_ptr(logits), B, T, V, logits.stride(0), logits.stride(1), _ptr(temperature), _ptr(top_p),
            ctypes.c_uint64(int(seed) & (2 ** 64 - 1)), _ptr(offset), _ptr(ids), ids.stride(0), _ptr(rows), _ptr(drop), _ptr(history),
            history.shape[1] if history is not None else 0, _ptr(length), _ptr(limit), _ptr(done), _ptr(steps), _ptr(accepted), eos_arr,
            len(eos), _ptr(status), _ptr(debug), _ptr(debug_w))
    with torch.cuda.device(logits.device):
        if filters is None:
            N.check(lib.mpig_aux_verify_sample(*args, _stream()), "mpig_aux_verify_sample")
        else:
            f = filters.native()
            N.check(lib.mpig_aux_verify_sample_filtered(*args, ctypes.byref(f), _stream()), "mpig_aux_verify_sample_filtered")
    return ids


PROMPT_BIT = -(1 << 31)   # bit 31 of a penalty-table entry, as int32


@dataclass
class SampleFilters:
    """The sampling filters of sample(..., filters=) and verify_sample(..., filters=) (mpig_sample_filters in
    include/magicpig_b200_aux.h states the rule): per-request device arrays of shape (B,) -- top_k int32 (<= 0: off), min_p fp32 in
    [0, 1] (0: off), repetition_penalty fp32 > 0 (1: off), presence_penalty and frequency_penalty fp32 in [-2, 2] (0: off) -- and the
    penalty table, (B, ld >= V) int32 or uint32 with contiguous rows: the low 31 bits of entry i count request b's emitted token i,
    bit 31 marks a token of its prompt (penalty_table() builds it).  The filtered calls increment the entries of the tokens they
    append."""
    top_k: torch.Tensor
    min_p: torch.Tensor
    repetition_penalty: torch.Tensor
    presence_penalty: torch.Tensor
    frequency_penalty: torch.Tensor
    table: torch.Tensor

    @classmethod
    def neutral(cls, B: int, V: int, device) -> "SampleFilters":
        """Every filter off and an empty table: the filtered calls then compute what the unfiltered ones do."""
        f32 = lambda v: torch.full((B,), v, dtype=torch.float32, device=device)  # noqa: E731
        return cls(torch.zeros((B,), dtype=torch.int32, device=device), f32(0.0), f32(1.0), f32(0.0), f32(0.0),
                   torch.zeros((B, V), dtype=torch.int32, device=device))

    def native(self) -> N.MpigSampleFilters:
        return N.MpigSampleFilters(self.top_k.data_ptr(), self.min_p.data_ptr(), self.repetition_penalty.data_ptr(),
                                   self.presence_penalty.data_ptr(), self.frequency_penalty.data_ptr(), self.table.data_ptr(),
                                   self.table.stride(0))


def check_filter_values(top_k=None, min_p=None, repetition_penalty=None, presence_penalty=None, frequency_penalty=None):
    """The value ranges of the filters, on host sequences (MagicPigError): min_p in [0, 1], repetition_penalty finite and > 0,
    presence / frequency penalties in [-2, 2]; top_k any integer (<= 0 is off)."""
    def floats(name, vals, ok, what):
        for v in vals:
            if not (isinstance(v, (int, float)) and math.isfinite(float(v)) and ok(float(v))):
                raise N.MagicPigError(f"{name}: every value must be {what}, got {v!r}")
    if top_k is not None:
        for v in top_k:
            if isinstance(v, bool) or not float(v).is_integer() or not -2 ** 31 <= int(v) < 2 ** 31:
                raise N.MagicPigError(f"top_k: every value must be an int32 integer, got {v!r}")
    if min_p is not None:
        floats("min_p", min_p, lambda v: 0.0 <= v <= 1.0, "in [0, 1]")
    if repetition_penalty is not None:
        floats("repetition_penalty", repetition_penalty, lambda v: v > 0.0, "finite and > 0")
    for name, vals in (("presence_penalty", presence_penalty), ("frequency_penalty", frequency_penalty)):
        if vals is not None:
            floats(name, vals, lambda v: -2.0 <= v <= 2.0, "in [-2, 2]")


def check_filters(filters, B: int, V: int, device, values: Optional[bool] = None):
    """The checks of a SampleFilters on any device (MagicPigError): types, dtypes, shapes, devices, the table's layout, and the
    values' ranges.  values=None checks the values unless the current stream is capturing a graph (reading them then would break
    the capture; the device takes a value outside its range as neutral)."""
    if not isinstance(filters, SampleFilters):
        raise N.MagicPigError(f"filters: expected a SampleFilters, got {type(filters).__name__}")
    _sample_chk(filters.top_k, torch.int32, (B,), "top_k", device)
    for name in ("min_p", "repetition_penalty", "presence_penalty", "frequency_penalty"):
        _sample_chk(getattr(filters, name), torch.float32, (B,), name, device)
    for name in ("top_k", "min_p", "repetition_penalty", "presence_penalty", "frequency_penalty"):
        if not getattr(filters, name).is_contiguous():
            raise N.MagicPigError(f"{name}: must be contiguous")
    t = filters.table
    if not isinstance(t, torch.Tensor) or t.dtype not in (torch.int32, torch.uint32):
        raise N.MagicPigError("table: expected an int32 or uint32 tensor")
    _sample_chk(t, t.dtype, None, "table", device)
    if t.dim() != 2 or t.shape[0] != B or t.shape[1] < V or t.stride(1) != 1 or t.stride(0) < V:
        raise N.MagicPigError(f"table: expected (B={B}, ld >= V={V}) with contiguous rows, got {tuple(t.shape)} strides {t.stride()}")
    if values is None:
        values = not (device.type == "cuda" and torch.cuda.is_current_stream_capturing())
    if values:
        check_filter_values(filters.top_k.tolist(), filters.min_p.tolist(), filters.repetition_penalty.tolist(),
                            filters.presence_penalty.tolist(), filters.frequency_penalty.tolist())


def penalty_table(prompts, V: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The penalty table at the start of a generation: zero counts and bit 31 set on each request's prompt tokens.  prompts: one
    1-D tensor (or sequence) of token ids per request, or a (B, P) tensor.  out: int32 / uint32 (B, ld >= V) with contiguous rows,
    written in place (None: a new int32 (B, V) tensor on the prompts' device).  Torch ops, once per generation.  Returns out."""
    rows = list(prompts.unbind(0)) if isinstance(prompts, torch.Tensor) and prompts.dim() == 2 else list(prompts)
    rows = [torch.as_tensor(p).reshape(-1) for p in rows]
    B = len(rows)
    if B < 1 or int(V) < 1:
        raise N.MagicPigError(f"penalty_table: need at least one prompt and V >= 1, got {B} prompts and V={V}")
    if out is None:
        out = torch.zeros((B, int(V)), dtype=torch.int32, device=rows[0].device)
    if not isinstance(out, torch.Tensor) or out.dtype not in (torch.int32, torch.uint32) or out.dim() != 2:
        raise N.MagicPigError("penalty_table: out must be an int32 or uint32 (B, ld) tensor")
    if out.shape[0] != B or out.shape[1] < V or out.stride(1) != 1:
        raise N.MagicPigError(f"penalty_table: out must be (B={B}, ld >= V={V}) with contiguous rows, got {tuple(out.shape)}")
    for b, p in enumerate(rows):
        if p.numel() and (p.dtype.is_floating_point or p.dtype == torch.bool):
            raise N.MagicPigError(f"penalty_table: prompt {b} must hold integer token ids, got {p.dtype}")
        if p.numel() and (int(p.min()) < 0 or int(p.max()) >= V):
            raise N.MagicPigError(f"penalty_table: prompt {b} holds ids outside [0, V={V})")
    view = out.view(torch.int32)
    view.zero_()
    for b, p in enumerate(rows):
        view[b].index_fill_(0, p.to(out.device, torch.int64), PROMPT_BIT)
    return out


def check_ngram_args(history, length, ids, T, g_min, g_max):
    """The argument checks of ngram_draft() on any device (no library call).  Raises MagicPigError."""
    if not isinstance(history, torch.Tensor) or history.dim() != 2:
        raise N.MagicPigError("history: expected a (B, n) tensor")
    dev = history.device
    _sample_chk(history, torch.int32, None, "history", dev)
    B = history.shape[0]
    if B < 1 or history.shape[1] < 1 or not history.is_contiguous():
        raise N.MagicPigError(f"history: expected a contiguous non-empty (B, n) tensor, got {tuple(history.shape)}")
    _sample_chk(length, torch.int32, (B,), "length", dev)
    if not length.is_contiguous():
        raise N.MagicPigError("length: must be contiguous")
    if not 1 <= int(T) <= MAX_VERIFY_TOKENS:
        raise N.MagicPigError(f"T={T} outside [1, {MAX_VERIFY_TOKENS}]")
    if not 1 <= int(g_min) <= int(g_max) <= MAX_NGRAM:
        raise N.MagicPigError(f"need 1 <= g_min <= g_max <= {MAX_NGRAM}, got g_min={g_min}, g_max={g_max}")
    _ids_chk(ids, B, int(T), dev)


def ngram_draft(history: torch.Tensor, length: torch.Tensor, ids: torch.Tensor, T: int, g_min: int = 1, g_max: int = 3) -> torch.Tensor:
    """Prompt-lookup drafts on the device (mpig_aux_ngram_draft, include/magicpig_b200_aux.h, states the rule): from the token
    history int32 (B, n) of device lengths int32 (B,), T - 1 drafts per request into ids[b, 1:T] (int64 (B, >= T)): the text after
    the most recent of the longest earlier matches (g_min .. g_max tokens) of the history's suffix, copied with overlap; the last
    token repeated when nothing matches.  Checked here before the call; capturable.  Returns ids."""
    check_ngram_args(history, length, ids, T, g_min, g_max)
    if history.device.type != "cuda":
        raise N.MagicPigError("ngram_draft runs on CUDA (sm_90a) only; there is no CPU path")
    lib = N.load()
    with torch.cuda.device(history.device):
        N.check(lib.mpig_aux_ngram_draft(_ptr(history), history.shape[0], history.shape[1], _ptr(length), _ptr(ids), ids.stride(0),
                                         int(T), int(g_min), int(g_max), _stream()), "mpig_aux_ngram_draft")
    return ids


# =================================================================================================
# Reference-named facades
# =================================================================================================
class LSH:
    """Mirror of `lsh.LSH` (library/lsh/lsh.cc:316-326) with HBM-resident tables."""

    def __init__(self, ctx: Optional[Context] = None, device: str = "cuda:0"):
        self.ctx = ctx
        self._own = ctx is None
        self._device = device

    def alloc(self, K: int, L: int, num_layers: int, num_attention_heads: int, num_key_value_heads: int,
              batch_size: int, max_length: int):
        """lsh.cc:44-91"""
        if self.ctx is None:
            self.ctx = Context(K, L, num_layers, num_attention_heads, num_key_value_heads, 128, batch_size, max_length,
                               device=self._device)
        self.ctx.set_option("save_mask", 1)

    def fill(self, layer_id: int, request_id: int, sorted_hash_code: torch.Tensor, sorted_indices: torch.Tensor):
        """lsh.cc:143-201"""
        self.ctx.lsh_fill(layer_id, request_id, sorted_hash_code.contiguous(), sorted_indices.contiguous())

    def build(self, layer_id: int, request_id: int, hash_code: torch.Tensor):
        """Device-side counting sort replacing `sort()` + fill (attnserver.py:186-193)."""
        self.ctx.lsh_build(layer_id, request_id, hash_code.contiguous())

    def fastfill(self, layer_id: int, request_id: int, hash_code: torch.Tensor):
        """lsh.cc:93-142: tables from UNSORTED per-key codes (Hkv, L, n).  Bound by the reference's pybind module but
        unfinished there (it counts buckets and never writes the table content); here it is the counting-sort build.
        int32 codes (the reference's dtype for this entry point) are narrowed to the int16 the build consumes."""
        if hash_code.dtype != torch.int16:
            hash_code = hash_code.to(torch.int16)
        self.build(layer_id, request_id, hash_code)

    def batch_retrieve(self, layer_id: int, query: torch.Tensor, results: torch.Tensor, nnz: torch.Tensor):
        """lsh.cc:210-241"""
        self.ctx.lsh_batch_retrieve(layer_id, query, results, nnz)

    def get_mask(self) -> torch.Tensor:
        """lsh.cc:308-314 (int8 view in the reference; values {0,1,2})"""
        return self.ctx.lsh_get_mask().view(torch.int8)

    def copy(self, query: torch.Tensor):
        """lsh.cc:203-207: a no-op in the reference too."""

    def clear(self):
        """lsh.cc:293-306"""
        self.ctx.clear()


class SparseAttentionServer:
    """Mirror of `sparse_attention_cpu.SparseAttentionServer` (sparse_attention.cc:1243-1263)."""

    def __init__(self, ctx: Optional[Context] = None, device: str = "cuda:0"):
        self.ctx = ctx
        self._device = device

    def alloc(self, num_layers: int, num_attention_heads: int, num_key_value_heads: int, head_dim: int,
              batch_size: int, max_length: int):
        """sparse_attention.cc:546-583"""
        if self.ctx is None:
            # tables are not used through this facade: K = L = 1 keeps them tiny
            self.ctx = Context(1, 1, num_layers, num_attention_heads, num_key_value_heads, head_dim, batch_size,
                               max_length, device=self._device)

    def fill(self, layer_id: int, request_id: int, k: torch.Tensor, v: torch.Tensor, kn: torch.Tensor):
        """sparse_attention.cc:601-627"""
        self.ctx.attn_fill(layer_id, request_id, k.contiguous(), v.contiguous(), kn.contiguous())

    def attention_wrapper(self, layer_id: int, K: int, L: int, output: torch.Tensor, max_value_expsum: torch.Tensor,
                          query: torch.Tensor, query_norm: torch.Tensor, ind: torch.Tensor, nnz: torch.Tensor):
        """sparse_attention.cc:629-745"""
        self.ctx.attention_wrapper(layer_id, K, L, output, max_value_expsum, query.contiguous(),
                                   query_norm.contiguous(), ind, nnz)

    # the reference exposes several spellings of the same computation (sparse_attention.cc:1246-1255)
    attention = attention_wrapper
    attention_bf16 = attention_wrapper
    attention_wrapper_bf16 = attention_wrapper
    scheduled_attention = attention_wrapper

    def get_key_cache(self, layer_id: int) -> torch.Tensor:
        return self.ctx.read_cache(layer_id, True, False, False)[0]

    def get_value_cache(self, layer_id: int) -> torch.Tensor:
        return self.ctx.read_cache(layer_id, False, True, False)[1]

    def get_key_norm(self, layer_id: int) -> torch.Tensor:
        return self.ctx.read_cache(layer_id, False, False, True)[2]

    def clear(self):
        """sparse_attention.cc:586-598"""
        self.ctx.clear()
