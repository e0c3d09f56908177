"""`LSHSparseAttnServer` -- drop-in for MagicPIG's `models/attnserver.py::LSHSparseAttnServer`.

Same constructor keywords and the same seven methods, with the same argument meaning, as the
reference class (models/attnserver.py:7-331) so that `models/llama.py` can construct and drive it
unchanged (`llama.py:91-93, 208, 264, 282-284, 292, 315, 357`):

    alloc_buffer(seq_len) / fill(layer, request, k, v, seq_len) / build_table(layer, request, seq_len)
    plan() / decode(q, k, v, layer) -> (B, 1, hidden) / clear()

What changes is where things live and run: the offloaded KV cache, the L hash tables and the
sink/local/generated window are resident in HBM inside a `magicpig_b200.ops.Context`, and a sparse
layer's decode is three hand-written sm_90a kernels (SimHash -> probe -> gather attention with the
window merge folded in) instead of a GPU->CPU->GPU round trip through OpenMP/AVX-512 operators.
There is no FlashInfer dependency and no CPU fallback.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from .ops import Context
from . import synth


def beam_sources(parents: torch.Tensor):
    """Where the new beams of a beam-search step live.  parents (B,) int: new beam i continues old beam parents[i], old beam j
    being held by request j.  Returns (src_of, request_of), both int32 (B,) on parents' device:
      request_of[i]  the request that holds new beam i: each chosen parent keeps its own request for its first child (in i order),
                     the other children take the requests of the unchosen parents in ascending order (a permutation);
      src_of         the map for LSHSparseAttnServer.reorder: src_of[request_of[i]] = parents[i].  Every source keeps its own
                     request, so src_of[src_of[b]] == src_of[b] by construction.
    Device torch ops only (B x B comparisons): no host synchronisation and no data-dependent shapes, so it can be captured."""
    p = parents.long().reshape(-1)
    B = p.numel()
    ar = torch.arange(B, device=p.device)
    same = p[:, None] == p[None, :]                                    # [i, j]: beams i and j have one parent
    first = ~(same & (ar[None, :] < ar[:, None])).any(dim=1)          # i is its parent's first child
    chosen = (p[None, :] == ar[:, None]).any(dim=1)                   # [r]: request r holds a parent
    free_rank = torch.cumsum((~chosen).long(), 0) - 1                 # rank of an unchosen request among the unchosen
    free = ((~chosen[None, :]) & (free_rank[None, :] == ar[:, None])).long()   # [k, r]: r is the k-th unchosen request
    free_req = (free * ar[None, :]).sum(dim=1)                        # the k-th unchosen request (k < their count)
    child_rank = (torch.cumsum((~first).long(), 0) - 1).clamp(min=0)  # rank of a later child among the later children
    request_of = torch.where(first, p, free_req[child_rank])
    src_of = torch.empty_like(p)
    src_of[request_of] = p
    return src_of.to(torch.int32), request_of.to(torch.int32)


PREFILL_DTYPES = (torch.bfloat16, torch.float16, torch.float32)


def check_prefill_args(q, k, v, num_attention_heads: int, num_key_value_heads: int, head_dim: int, causal: bool = True,
                       kv_layout: str = "NHD"):
    """The refusals of LSHSparseAttnServer.prefill_attention, before anything runs: ValueError unless causal, kv_layout "NHD",
    q (q_len, Hq, d) and k / v (kv_len, Hkv, d) with the server's per-rank head counts, 1 <= q_len <= kv_len, k and v of one shape,
    and floating dtypes (bf16, fp16 or fp32).  Shape and dtype checks only: the tensors may live anywhere."""
    if not causal:
        raise ValueError("prefill_attention computes causal attention only (causal=False is not supported)")
    if kv_layout != "NHD":
        raise ValueError(f"prefill_attention takes the NHD layout only, got kv_layout={kv_layout!r}")
    Hq, Hkv, d = num_attention_heads, num_key_value_heads, head_dim
    if q.dim() != 3 or tuple(q.shape[1:]) != (Hq, d):
        raise ValueError(f"q must be (q_len, {Hq}, {d}), got {tuple(q.shape)}")
    if k.dim() != 3 or tuple(k.shape[1:]) != (Hkv, d):
        raise ValueError(f"k must be (kv_len, {Hkv}, {d}), got {tuple(k.shape)}")
    if tuple(v.shape) != tuple(k.shape):
        raise ValueError(f"v must have k's shape {tuple(k.shape)}, got {tuple(v.shape)}")
    if not 1 <= q.shape[0] <= k.shape[0]:
        raise ValueError(f"need 1 <= q_len <= kv_len, got q_len={q.shape[0]}, kv_len={k.shape[0]}")
    for name, t in (("q", q), ("k", k), ("v", v)):
        if t.dtype not in PREFILL_DTYPES:
            raise ValueError(f"{name} must be bf16, fp16 or fp32, got {t.dtype}")


class LSHSparseAttnServer:
    def __init__(self,
                 config,
                 K: int = 10,
                 L: int = 150,
                 batch_size: int = 1,
                 num_sink_tokens: int = 4,
                 num_local_tokens: int = 64,
                 generation_buffer: int = 256,
                 max_length: int = 8192,
                 dense_layers: Sequence[int] = (0, 16, 32, 48, 64),
                 device: str = "cuda:0",
                 dtype=torch.bfloat16,
                 hash_func: Optional[torch.Tensor] = None,
                 table_build: str = "device",
                 key_hash: str = "tcgen05",
                 num_key_value_heads: Optional[int] = None,
                 num_attention_heads: Optional[int] = None,
                 max_query_tokens: int = 1,
                 num_contexts: Optional[int] = None,
                 dense_tail_rows: Optional[int] = None,
                 shared_spill: bool = False,
                 max_chunk_tokens: int = 0) -> None:
        """Keywords up to `dtype` are the reference's (attnserver.py:9-20).  Extras:
        hash_func   inject the (d, K*L) bf16 projection (the reference draws it unseeded, :55);
        table_build "device" = counting sort on the GPU (mpig_lsh_build); "sorted" = the reference's
                    `sort()` + LSH.fill route (attnserver.py:186-193) with the fill done on the GPU;
        key_hash    "tcgen05" (the name of the first target's tensor cores, kept for compatibility) = key-side SimHash GEMM +
                    sign pack in one tensor-core kernel (mpig_hash_keys, wgmma on sm_90a);
                    "torch" = the reference's chunked `matmul(...).gt(0)` + pack glue (attnserver.py:159-168);
        num_*_heads per-rank head counts under KV-head tensor parallelism (attnserver_dist.py:252-254);
        max_query_tokens  largest number of draft tokens a verification step may check (plan(num_tokens), decode of q_len > 1,
                    rewind); 1 = single-token decoding only.
        num_contexts number of contexts (sampled stores + hash tables) the batch holds, 1..batch_size; None = batch_size.
                    Request b starts on context b mod num_contexts; fork() and bind() change that.
        dense_tail_rows R > 0: the dense layers' prompt rows are kept once per context too, and each request holds only the R
                    rows it adds after its prompt (needs num_contexts < batch_size); None = a full dense cache per request.
        shared_spill  requests that share a context may spill_window() into it (needs num_contexts < batch_size <= 32): each
                    spilled token is private to the request that spilled it and to requests later forked from it.  Size max_length
                    for the prompt plus every request's spilled tokens, or call compact() after spills to free the
                    tokens no request sees any more and size it for the live ones.
        max_chunk_tokens  largest T of a chunk step (plan_chunk(T): T new prompt tokens per request, attended exactly); 0 = none.
        """
        self.K, self.L = K, L
        self.config = config
        self.length = num_sink_tokens + num_local_tokens + generation_buffer
        self.max_length = max_length
        self.device = torch.device(device)
        self.dtype = dtype
        self.num_layers = config.num_hidden_layers
        self.batch_size = batch_size
        self.num_key_value_heads = num_key_value_heads or config.num_key_value_heads
        self.num_attention_heads = num_attention_heads or config.num_attention_heads
        self.head_dim = config.hidden_size // config.num_attention_heads
        self.hidden_size = self.num_attention_heads * self.head_dim  # per rank
        self.dense_layers = [l for l in dense_layers if l < self.num_layers]
        self.num_sink_tokens = num_sink_tokens
        self.num_local_tokens = num_local_tokens
        self.num_key_value_groups = self.num_attention_heads // self.num_key_value_heads
        self.table_build = table_build
        if key_hash not in ("tcgen05", "torch"):
            raise ValueError(f"key_hash must be 'tcgen05' or 'torch', got {key_hash!r}")
        self.key_hash = key_hash
        self.chunk_size = 8192

        self.ctx = Context(K, L, self.num_layers, self.num_attention_heads, self.num_key_value_heads, self.head_dim,
                           batch_size, max_length, num_sink_tokens, num_local_tokens, generation_buffer,
                           dense_layers=self.dense_layers, alloc_dense_kv=True, device=self.device,
                           max_query_tokens=max_query_tokens, num_contexts=num_contexts or 0,
                           dense_tail_rows=dense_tail_rows or 0, shared_spill=shared_spill)
        if max_chunk_tokens > 0:
            self.ctx.reserve_chunk_tokens(max_chunk_tokens)
        if hash_func is None:
            hash_func = torch.randn((self.head_dim, K * L), device=self.device, dtype=torch.bfloat16)  # attnserver.py:55
        self.hash_func = hash_func.to(device=self.device, dtype=torch.bfloat16).contiguous()
        self.ctx.set_hash_func(self.hash_func)
        self.avg_k = [torch.zeros(batch_size, self.num_key_value_heads, 1, self.head_dim, device=self.device,
                                  dtype=torch.bfloat16) for _ in range(self.num_layers)]
        # key codes of the layer whose table is being built (one layer in flight, as the reference)
        self.hash_code_buffer = torch.zeros((self.num_key_value_heads, L, max_length), dtype=torch.int16, device=self.device)
        self._out = {}   # layer (one token) or (layer, T) (T-token steps) -> decode output buffer (allocated on first use)
        self._tree_stage = {}   # staging of host-side tree parents / accepted paths / rewind counts, per (name, shape)

    # ------------------------------------------------------------------------------------------
    def alloc_buffer(self, seq_len: int):
        """attnserver.py:108-110 allocates pinned host sort buffers; nothing leaves the GPU here."""
        self._offload_len = seq_len - self.num_sink_tokens - self.num_local_tokens

    def fill(self, layer_idx: int, request_id: int, key_cache: torch.Tensor, value_cache: torch.Tensor, seq_len: int):
        """attnserver.py:112-175.  key_cache/value_cache (>=seq_len, Hkv, d) in NHD layout."""
        if layer_idx in self.dense_layers:
            kc = key_cache.to(torch.bfloat16).contiguous()
            vc = value_cache.to(torch.bfloat16).contiguous()
            self.ctx.dense_fill(layer_idx, request_id, kc, vc, seq_len)
            return
        ns, nl = self.num_sink_tokens, self.num_local_tokens
        key_cache = key_cache.to(torch.bfloat16)
        value_cache = value_cache.to(torch.bfloat16)
        key = torch.cat([key_cache[:ns], key_cache[seq_len - nl:seq_len]], dim=0).transpose(0, 1)
        value = torch.cat([value_cache[:ns], value_cache[seq_len - nl:seq_len]], dim=0).transpose(0, 1)
        offload_key = key_cache[ns:seq_len - nl].transpose(0, 1).contiguous()      # (Hkv, n, d)
        offload_value = value_cache[ns:seq_len - nl].transpose(0, 1).contiguous()
        avg_k = offload_key.mean(dim=1, keepdim=True)                                # attnserver.py:142
        key = key - avg_k
        offload_key = offload_key - avg_k
        kn = offload_key.norm(p=2, dim=-1).float()                                   # attnserver.py:146 (bf16-rounded)
        self.avg_k[layer_idx][request_id] = avg_k
        n = offload_key.shape[1]
        # key-side SimHash (attnserver.py:159-168): tensor-core GEMM with the sign-pack epilogue (csrc/keyhash.cu); the torch
        # GEMM + pack glue stays selectable (key_hash="torch") as the cross-check the tests use
        if self.key_hash == "tcgen05":
            self.hash_code_buffer[:, :, :n].copy_(self.ctx.hash_keys(offload_key.contiguous()))
        else:
            self.hash_code_buffer[:, :, :n].copy_(synth.hash_keys(offload_key, self.hash_func, self.K, self.L, self.chunk_size))
        self.ctx.attn_fill(layer_idx, request_id, offload_key, offload_value.contiguous(), kn.contiguous())
        self.ctx.window_fill(layer_idx, request_id, avg_k.reshape(self.num_key_value_heads, self.head_dim).contiguous(),
                             key.contiguous(), value.contiguous())

    def build_table(self, layer_idx: int, request_id: int, seq_len: int):
        """attnserver.py:178-193."""
        if layer_idx in self.dense_layers:
            return
        n = seq_len - self.num_sink_tokens - self.num_local_tokens
        codes = self.hash_code_buffer[:, :, :n]
        if self.table_build == "sorted":
            sorted_codes, sorted_idx = codes.sort()
            self.ctx.lsh_fill(layer_idx, request_id, sorted_codes.contiguous(), sorted_idx.int().contiguous())
        else:
            self.ctx.lsh_build(layer_idx, request_id, codes.contiguous())

    def fork(self, src_request: int, dst_requests):
        """Not in the reference.  Each request of dst_requests (an int or a sequence) continues from src_request's state: it
        decodes over src_request's context (no copy of the sampled store or the tables) and gets a copy of its sink + local +
        generated window, its dense-layer KV and its lengths.  The usual way to serve n answers to one prompt, or several
        questions about one document: fill and build one request, then fork it.  Requests sharing a context generate at most
        generation_buffer tokens (spill_window() refuses them) unless the server was made with shared_spill=True: then each dst
        sees exactly the tokens src spilled before the fork, and each request's later spills stay its own.  Needs num_contexts <
        batch_size."""
        for dst in ([dst_requests] if isinstance(dst_requests, int) else dst_requests):
            self.ctx.fork(src_request, dst)
            for a in self.avg_k:
                a[dst].copy_(a[src_request])

    def reorder(self, src_of: torch.Tensor):
        """Not in the reference.  Request b continues request src_of[b]'s sequence: fork(src_of[b], b) for every b with
        src_of[b] != b, done on the device (the server's avg_k copies are gathered with device ops too).  src_of: device int32
        (B,) whose sources are fixed points (src_of[src_of[b]] == src_of[b]); beam_sources() builds one from a beam step's
        parents.  CUDA-graph capturable.  Needs num_contexts < batch_size."""
        self.ctx.reorder(src_of)
        idx = src_of.long()
        for a in self.avg_k:
            a.copy_(a.index_select(0, idx))

    def bind(self, request: int, context: int):
        """Not in the reference.  Bind `request` to context slot `context` (0 <= context < num_contexts); fill() and
        build_table() of the request then write that context, which every request bound to it reads.  With shared_spill the
        request sees none of the tokens spilled into a context until it spills again."""
        self.ctx.bind(request, context)

    def plan(self, num_tokens: int = 1, parents=None):
        """attnserver.py:196-224.  num_tokens > 1: a verification step of that many tokens per request (the decode calls of the
        step then take q_len = num_tokens); rewind() afterwards drops the rejected ones.  With `parents` the step is a token tree
        of num_tokens nodes: parents[b][t] is node t's parent (parents[b][0] = -1, 0 <= parents[b][t] < t), a (T,) list applies to
        every request, a device int32 (B, T) tensor goes through without a copy (capturable).  Node t attends to the context, its
        ancestors and itself; accept() afterwards commits one root path per request."""
        if parents is None:
            self.ctx.plan(num_tokens)
            return
        T = int(num_tokens)
        self.ctx.plan(T, parents=self._stage_int32("parents", parents, (self.batch_size, T)))

    def plan_chunk(self, num_tokens: int):
        """Not in the reference.  A chunk step: num_tokens (<= max_chunk_tokens) new prompt tokens per request -- a follow-up turn, or
        a forked request's question.  The decode calls of the step take q_len = num_tokens on sparse and dense layers alike, and token t
        gets exact causal attention over the whole context (the request's store and window, or its dense rows) and the chunk's tokens up
        to t.  rewind() afterwards keeps a ragged prefix per request; spill_window() folds the chunk into the store."""
        self.ctx.plan_chunk(int(num_tokens))

    def accept(self, nodes, num_accepted):
        """Not in the reference.  Commits the root path nodes[b][0 .. num_accepted[b]) of the pending step (tree or chain): the
        path's K/V rows become the step's first rows in every layer and the lengths grow by num_accepted[b] only.  nodes: (T,) list
        (every request), (B, <= T) sequences or a device int32 (B, T) tensor; num_accepted: an int, B ints or a device int32 (B,)
        tensor.  Device tensors go through without a copy (capturable: acceptance can be decided on the GPU)."""
        T = self.ctx.pending_tokens
        if isinstance(num_accepted, int):
            num_accepted = [num_accepted] * self.batch_size
        self.ctx.accept(self._stage_int32("nodes", nodes, (self.batch_size, T)),
                        self._stage_int32("count", num_accepted, (self.batch_size,)))

    def _stage_int32(self, name: str, x, shape) -> torch.Tensor:
        """A device int32 tensor of `shape` for x: device tensors as they are, host sequences copied into a staging buffer
        (a per-request sequence shorter than the row is padded with zeros; one row broadcasts to every request)."""
        if isinstance(x, torch.Tensor) and x.is_cuda:
            return x.to(torch.int32).reshape(shape).contiguous()
        rows = [list(r) for r in x] if len(shape) == 2 and len(x) and not isinstance(x[0], int) else None
        host = torch.zeros(shape, dtype=torch.int32)
        if len(shape) == 1:
            host[:] = torch.as_tensor(list(x), dtype=torch.int32)
        elif rows is None:
            host[:, :len(x)] = torch.as_tensor(list(x), dtype=torch.int32)
        else:
            for b, r in enumerate(rows):
                host[b, :len(r)] = torch.as_tensor(r, dtype=torch.int32)
        buf = self._tree_stage.get((name, shape))
        if buf is None:
            buf = self._tree_stage[(name, shape)] = torch.zeros(shape, dtype=torch.int32, device=self.device)
        buf.copy_(host)
        return buf

    def rewind(self, num_rejected):
        """Not in the reference.  Drops the last `num_rejected` tokens of the pending verification step: an int (every request),
        a sequence of B ints, or a device int32 (B,) tensor (capturable: acceptance can be decided on the GPU)."""
        if isinstance(num_rejected, int):
            num_rejected = [num_rejected] * self.batch_size
        self.ctx.rewind(self._stage_int32("drop", num_rejected, (self.batch_size,)))

    def spill_window(self, keep: Optional[int] = None) -> torch.Tensor:
        """Not in the reference.  Moves the oldest generated tokens of every sparse layer's window into the sampled store and
        the hash tables, keeping the newest `keep` (default num_local_tokens) in the window, so that a generation can run past
        generation_buffer tokens.  Call it between tokens, never inside a captured step (it synchronises); plan() does not
        spill on its own.  Returns the spilled token count per request, int32 (B,) on the host.  Requests that share a context
        may spill only with shared_spill=True; their spilled tokens then go to the shared context but each request samples only
        its own (and those inherited through fork())."""
        return self.ctx.spill_window(keep)

    def compact(self, context: Optional[int] = None) -> torch.Tensor:
        """Not in the reference.  With shared_spill=True, frees the spilled tokens of a context (None: every context) that no
        request sees any more: those of a request that fork() overwrote, that a beam step's reorder dropped, that bind() moved
        away, or that was retired.  Every request keeps sampling exactly the tokens it sampled before.  Call it between tokens
        when spill_window() would exceed max_length (so max_length needs to hold the prompt plus the live spilled tokens only),
        for example after each spill of a beam search or after re-forking questions from one prompt.  To retire a finished
        request, bind() it to its own context first: its spilled tokens then die.  It synchronises, so it is never part of a
        captured step, but a step captured before it stays valid.  Returns the tokens freed per context, int32
        (num_contexts,) on the host (zeros without shared_spill)."""
        return self.ctx.compact(context)

    def decode(self, query_states: torch.Tensor, key_states: torch.Tensor, value_states: torch.Tensor, layer_idx: int):
        """attnserver.py:228-312.  q (B,Hq,1,d), k/v (B,Hkv,1,d) -> (B, 1, Hq*d).  In a verification step of T tokens (plan(T)):
        q (B,Hq,T,d), k/v (B,Hkv,T,d) -> (B, T, Hq*d), token t attending causally to the tokens before it."""
        T = query_states.shape[2]
        if self.ctx.pending_chunk:
            return self._decode_tokens(query_states, key_states, value_states, layer_idx, T, chunk=True)
        if T > 1:
            return self._decode_tokens(query_states, key_states, value_states, layer_idx, T)
        q = query_states.to(torch.bfloat16).contiguous()
        k = key_states.to(torch.bfloat16).contiguous()
        v = value_states.to(torch.bfloat16).contiguous()
        # one output buffer per layer, allocated on first use: a layer's output is consumed before that layer decodes the next
        # token, so decode() allocates nothing in steady state (and is CUDA-graph capturable with static addresses)
        out = self._out.get(layer_idx)
        if out is None:
            out = self._out[layer_idx] = torch.empty((self.batch_size, self.num_attention_heads * self.head_dim), dtype=torch.bfloat16,
                                                     device=self.device)
        if layer_idx in self.dense_layers:
            self.ctx.dense_decode(layer_idx, q, k, v, out)
        else:
            self.ctx.decode(layer_idx, q, k, v, out)
        return out.reshape(self.batch_size, 1, self.num_attention_heads * self.head_dim).to(query_states.dtype)

    def _decode_tokens(self, query_states, key_states, value_states, layer_idx: int, T: int, chunk: bool = False):
        # (B, H, T, d) -> the (B, T, H, d) layout of the T-token entry points
        q = query_states.to(torch.bfloat16).transpose(1, 2).contiguous()
        k = key_states.to(torch.bfloat16).transpose(1, 2).contiguous()
        v = value_states.to(torch.bfloat16).transpose(1, 2).contiguous()
        out = self._out.get((layer_idx, T))
        if out is None:
            out = self._out[(layer_idx, T)] = torch.empty((self.batch_size, T, self.num_attention_heads * self.head_dim),
                                                          dtype=torch.bfloat16, device=self.device)
        if chunk:
            self.ctx.chunk_attend(layer_idx, T, q, k, v, out)
        elif layer_idx in self.dense_layers:
            self.ctx.dense_decode_tokens(layer_idx, T, q, k, v, out)
        else:
            self.ctx.decode_tokens(layer_idx, T, q, k, v, out)
        return out.to(query_states.dtype)

    def prefill_attention(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = True,
                          allow_fp16_qk_reduction: bool = False, kv_layout: str = "NHD") -> torch.Tensor:
        """Not in the reference's server: the prefill attention the reference calls FlashInfer for (llama.py:250-257,
        flashinfer.prefill.single_prefill_with_kv_cache), with the same keywords, so that call becomes
        self.attention_server.prefill_attention(...).  q (q_len, Hq, d), k / v (kv_len, Hkv, d) NHD -> (q_len, Hq, d) in q's dtype:
        exact causal softmax attention, query i seeing keys [0, kv_len - q_len + i] (the chunk's queries are the last q_len
        positions), scale 1/sqrt(d).  Inputs are rounded to bf16 for the tensor cores; the product, the softmax and P.V accumulate
        in fp32, so allow_fp16_qk_reduction is accepted and has no effect.  causal=False or another kv_layout raises ValueError.
        Uses no server state (any layer, before or after fill); capturable."""
        check_prefill_args(q, k, v, self.num_attention_heads, self.num_key_value_heads, self.head_dim, causal, kv_layout)
        out = self.ctx.prefill_attend(q.to(torch.bfloat16).contiguous(), k.to(torch.bfloat16).contiguous(),
                                      v.to(torch.bfloat16).contiguous())
        return out.to(q.dtype)

    def clear(self):
        """attnserver.py:314-331."""
        for a in self.avg_k:
            a.zero_()
        self.hash_code_buffer.zero_()
        self.ctx.clear()
