"""Minimal Llama decode loop around `LSHSparseAttnServer` -- the CALLER side of the hot path.

The reference's caller is `models/llama.py` (hand-rolled Llama, `LLM.inference` :288-301,
`layer_compute` :185-220).  It needs HF checkpoints, FlashInfer and network access, none of which
exist on the benchmark box, so bench.py drives the attention server with this stand-in instead:
same per-layer sequence (RMSNorm -> q,k,v projections -> RoPE -> attention_server.decode -> wo ->
residual -> RMSNorm -> gated MLP -> residual), random-init weights of the named architecture,
library GEMMs (cuBLAS through torch).  Only the attention server is product code; everything in
this file is harness.

Context is synthetic by default: instead of a 98K-token prefill the per-layer K/V caches are filled with
seeded random tensors through the server's own `fill()` / `build_table()` (the reference's prefill-time
API), so tables, key norms, centring and the sink/local window are all produced by the real path.
`prefill()` is the real thing for one request: the forward of a prompt's token ids, with prefill
attention on the server's tensor-core kernel (`prefill_attention`), into the same fill()/build_table().
"""
from __future__ import annotations

import ctypes
import math
import os
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from . import _native as N
from . import ops, tp
from .attnserver import LSHSparseAttnServer, beam_sources


@dataclass
class LlamaShape:
    name: str = "Llama-3.1-8B-Instruct"
    num_hidden_layers: int = 32
    hidden_size: int = 4096
    intermediate_size: int = 14336
    num_attention_heads: int = 32
    num_key_value_heads: int = 8
    vocab_size: int = 128256
    rope_theta: float = 500000.0
    rms_norm_eps: float = 1e-5
    eos_token_ids: tuple = (128001, 128008, 128009)   # generate() stops a request at these ids (Llama-3.1's end-of-text ids)

    @property
    def head_dim(self):
        return self.hidden_size // self.num_attention_heads


LLAMA31_8B = LlamaShape()
LLAMA31_70B = LlamaShape("Llama-3.1-70B-Instruct", 80, 8192, 28672, 64, 8, 128256, 500000.0, 1e-5)


def rope_tables(theta: float, d: int, rows: int, device) -> tuple[torch.Tensor, torch.Tensor]:
    """The (rows, d) bf16 cos / sin tables of rotate-half RoPE for positions 0 .. rows - 1 (llama.py:111-124)."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, d, 2, device=device, dtype=torch.float32) / d))
    t = torch.arange(rows, device=device, dtype=torch.float32)
    freqs = torch.outer(t, inv_freq)
    emb = torch.cat([freqs, freqs], dim=-1)
    return emb.cos().to(torch.bfloat16), emb.sin().to(torch.bfloat16)


def plan_turn_chunks(lengths, t_max: int, room: int):
    """The chunk steps that feed a turn of lengths[b] tokens to request b: a list of (start, T, drop) with T <= min(t_max, room) tokens
    from position `start` of the turn, drop[b] = the tokens of the step past request b's length (rewound after it).  room = the window
    rows free after a spill (generation_buffer).  Pure host arithmetic."""
    step = min(int(t_max), int(room))
    if step < 1:
        raise ValueError(f"no room for a chunk: t_max={t_max}, room={room}")
    lengths = [int(n) for n in lengths]
    if any(n < 0 for n in lengths):
        raise ValueError(f"negative turn length in {lengths}")
    total = max(lengths, default=0)
    plan = []
    for start in range(0, total, step):
        T = min(step, total - start)
        plan.append((start, T, [T - min(max(n - start, 0), T) for n in lengths]))
    return plan


def plan_prefill_chunks(P: int, chunk_size: int, num_sink: int, num_local: int, max_length: int):
    """The (start, end) row ranges of the prompt chunks of a P-token prefill (llama.py:310-313: chunks of chunk_size, the last one
    ending at P).  Refuses (ValueError) a prompt the sparse layers cannot hold, P <= num_sink + num_local (nothing left to sample) or
    P > max_length, and chunk_size < 1.  Pure host arithmetic."""
    P, chunk_size = int(P), int(chunk_size)
    if chunk_size < 1:
        raise ValueError(f"chunk_size must be >= 1, got {chunk_size}")
    if P <= num_sink + num_local:
        raise ValueError(f"a prompt of {P} tokens does not reach past the sink + local window ({num_sink} + {num_local})")
    if P > max_length:
        raise ValueError(f"a prompt of {P} tokens exceeds max_length {max_length}")
    return [(start, min(start + chunk_size, P)) for start in range(0, P, chunk_size)]


GREEDY_TEMPERATURE = 0.1   # llama.py:340-343: below this temperature the reference takes the argmax


def per_request(value, B: int, name: str) -> list:
    """A scalar or a length-B sequence of floats -> B floats (ValueError otherwise)."""
    if isinstance(value, torch.Tensor):
        value = value.tolist()
    if isinstance(value, (int, float)):
        return [float(value)] * B
    vals = [float(v) for v in value]
    if len(vals) != B:
        raise ValueError(f"{name}: expected a scalar or {B} values, got {len(vals)}")
    return vals


def generate_prompts(prompt, B: int, num_contexts: int):
    """generate()'s prompt argument -> (list of 1-D prompts, shared): one tensor is every request's prompt; a list holds one prompt
    per request and needs one context per request.  Pure host checks (ValueError)."""
    if isinstance(prompt, torch.Tensor):
        p = prompt.reshape(-1) if prompt.dim() == 2 and prompt.shape[0] == 1 else prompt
        if p.dim() != 1:
            raise ValueError(f"prompt: expected (P,) token ids, got shape {tuple(prompt.shape)}")
        return [p] * B, True
    prompts = [torch.as_tensor(p).reshape(-1) for p in prompt]
    if len(prompts) != B:
        raise ValueError(f"prompt: expected one tensor or {B} prompts, got {len(prompts)}")
    if num_contexts < B:
        raise ValueError(f"B different prompts need one context per request ({num_contexts} contexts for {B} requests)")
    return prompts, False


def check_generate_args(lengths, max_new_tokens: int, check_every: int, eos, max_length: int, num_sink: int, num_local: int,
                        chunk_size: int, generation_buffer: int, can_spill: bool, *, B: int = 1, filters=None):
    """generate()'s refusals before anything is written (ValueError): max_new_tokens and check_every >= 1, at most 8 EOS ids,
    every prompt one the prefill takes with P + max_new_tokens <= max_length, and no spill needed where the server cannot spill
    (requests sharing a context without shared_spill).  filters: a dict of the sampling filters (top_k, min_p,
    repetition_penalty, presence_penalty, frequency_penalty), each a scalar or B values, refused outside their ranges
    (see filter_values).  Pure host arithmetic."""
    if filters is not None:
        filter_values(B, **filters)
    if int(max_new_tokens) < 1:
        raise ValueError(f"max_new_tokens must be >= 1, got {max_new_tokens}")
    if int(check_every) < 1:
        raise ValueError(f"check_every must be >= 1, got {check_every}")
    if len(eos) > ops.MAX_EOS_IDS:
        raise ValueError(f"at most {ops.MAX_EOS_IDS} EOS ids, got {len(eos)}")
    for P in lengths:
        plan_prefill_chunks(P, chunk_size, num_sink, num_local, max_length)
        if P + int(max_new_tokens) > max_length:
            raise ValueError(f"a prompt of {P} tokens + {max_new_tokens} new tokens exceeds max_length {max_length}")
    if int(max_new_tokens) - 1 > generation_buffer and not can_spill:
        raise ValueError(f"{max_new_tokens} new tokens need window spills, which requests sharing a context cannot do without "
                         "shared_spill")


def check_spec_args(lengths, max_new_tokens: int, draft_tokens: int, ngram, max_query_tokens: int, generation_buffer: int,
                    max_length: int, dense_tail_rows: int, can_spill: bool):
    """generate(draft_tokens=k)'s refusals beyond check_generate_args' (ValueError): k + 1 verification rows must fit
    max_query_tokens and the window (generation_buffer); P + max_new_tokens + k <= max_length for every prompt and, with
    dense_tail_rows R > 0, max_new_tokens + k <= R (a request holds at most P + max_new_tokens - 1 rows, also after it ends,
    and a step adds k + 1 before its rewind); no spill where the server cannot spill (requests sharing a context without
    shared_spill): the max_new_tokens - 1 replays must fit spec_spill_every(generation_buffer, k); and ngram = (g_min, g_max)
    needs 1 <= g_min <= g_max <= 8.  Pure host arithmetic."""
    k = int(draft_tokens)
    if k < 0:
        raise ValueError(f"draft_tokens must be >= 0, got {draft_tokens}")
    if k + 1 > max_query_tokens:
        raise ValueError(f"draft_tokens={k} needs max_query_tokens >= {k + 1} (the runner has {max_query_tokens})")
    if k + 1 > generation_buffer:
        raise ValueError(f"draft_tokens={k} needs generation_buffer >= {k + 1} (got {generation_buffer})")
    for P in lengths:
        if P + int(max_new_tokens) + k > max_length:
            raise ValueError(f"a prompt of {P} tokens + {max_new_tokens} new tokens + {k} drafts exceeds max_length {max_length}")
    if dense_tail_rows and int(max_new_tokens) + k > dense_tail_rows:
        raise ValueError(f"{max_new_tokens} new tokens with {k} drafts need {int(max_new_tokens) + k} dense tail rows "
                         f"(dense_tail_rows={dense_tail_rows})")
    if not can_spill and int(max_new_tokens) - 1 > spec_spill_every(generation_buffer, k):
        raise ValueError(f"{max_new_tokens} new tokens with {k} drafts need window spills (every "
                         f"{spec_spill_every(generation_buffer, k)} steps), which requests sharing a context cannot do without "
                         "shared_spill")
    g_min, g_max = (int(g) for g in ngram)
    if not 1 <= g_min <= g_max <= ops.MAX_NGRAM:
        raise ValueError(f"ngram=(g_min, g_max) needs 1 <= g_min <= g_max <= {ops.MAX_NGRAM}, got {tuple(ngram)}")


FILTER_NEUTRAL = dict(top_k=0, min_p=0.0, repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0)


def filter_values(B: int, **filters) -> dict:
    """The sampling filters given (None: not given) as B host values each, checked against their ranges (ValueError): top_k
    integers (<= 0: off), min_p in [0, 1], repetition_penalty finite and > 0, presence / frequency penalties in [-2, 2]."""
    out = {}
    for name, val in filters.items():
        if name not in FILTER_NEUTRAL:
            raise TypeError(f"unknown sampling filter {name!r}")
        if val is None:
            continue
        vals = per_request(val, B, name)
        if name == "top_k":
            if any(not float(v).is_integer() for v in vals):
                raise ValueError(f"top_k: expected integers, got {vals}")
            vals = [int(v) for v in vals]
        try:
            ops.check_filter_values(**{name: vals})
        except N.MagicPigError as e:
            raise ValueError(str(e)) from None
        out[name] = vals
    return out


def spec_spill_every(generation_buffer: int, draft_tokens: int) -> int:
    """Replays of the speculative graph between window spills: each keeps at most k + 1 rows and holds k + 1 during its step, so
    floor(generation_buffer / (k + 1)) replays fit the window with no device read to schedule the spill."""
    return int(generation_buffer) // (int(draft_tokens) + 1)


class LlamaDecodeRunner:
    # The CUDA-core GEMV issues 24*rows + 16 instructions per KB of weights per warp; at the HBM rate an SM has ~23 clocks per
    # KB (4 issue slots each), so it streams at the memory rate for rows <= 2 and is ALU-bound beyond (measured at rows = 8:
    # 9.6 ms per step).  Larger decode batches go through the library GEMM (tensor cores).
    GEMV_MAX_ROWS = 2

    def __init__(self, shape: LlamaShape, K: int, L: int, batch_size: int, max_length: int, device: str = "cuda:0",
                 seed: int = 0, generation_buffer: int = 256, dense_layers=(0, 16, 32, 48, 64), num_layers: int | None = None,
                 tp_rank: int = 0, tp_world: int = 1, tp_group=None, fused: bool = True, tp_mode: str = "ag",
                 tp_transport: str = "nccl", max_query_tokens: int = 1, num_contexts: int | None = None,
                 dense_tail_rows: int | None = None, shared_spill: bool = False, max_chunk_tokens: int = 0):
        """tp_mode (only with tp_world > 1; see magicpig_b200/tp.py):
             "ag"        attention sharded by KV head, one all-gather of head outputs per layer, wo / MLP replicated (north-star)
             "megatron"  + wo row-split, gate/up column-split, down row-split, two all-reduces per layer (llama_dist.py:49-70)
           tp_transport: "nccl" (torch.distributed collectives, captured in the CUDA graph) or "peer" (stores into the peers'
           buffers over NVLink: from the attention epilogue for "ag", one-shot all-reduce kernels for "megatron";
           magicpig_b200/peer.py).
           max_query_tokens: largest T of step_tokens(T) (verification steps of speculative decoding; 1 = step() only).
           num_contexts: contexts (sampled stores + hash tables) the batch holds; None = one per request.
           dense_tail_rows: R > 0 keeps the dense layers' prompt once per context, R rows per request after it; None = a full
           dense cache per request.
           shared_spill: requests forked from one prompt may spill their windows into the shared context (spill_window()), each
           seeing only its own spilled tokens; needs num_contexts < batch_size <= 32.
           max_chunk_tokens: largest chunk step extend() feeds at once (0 = extend() unavailable)."""
        assert tp_mode in ("ag", "megatron") and tp_transport in ("nccl", "peer")
        self.tp_mode, self.tp_transport = tp_mode, tp_transport
        self.shape = shape
        self.fused = fused
        self.use_gemv = os.environ.get("MPIG_GEMV", "1") != "0"   # decode linear layers through mpig_aux_gemv (fused step only)
        # PDL on the two edges around the attention kernel (include/magicpig_b200_aux.h: mpig_aux_set_pdl)
        # (measured on the full step, round 2: bit 0 alone -0.05 ms per token, bit 1 +0.08 ms: the parked o-projection CTAs pile
        # up on the 20 SMs the attention grid leaves free)
        N.load().mpig_aux_set_pdl(int(os.environ.get("MPIG_AUX_PDL", "1")))
        self.skip_sparse = os.environ.get("MPIG_SKIP_ATTN", "0") == "1"   # measurement aid: the step WITHOUT the sparse layers' attention
        # measurement aid (bench.py sets it on a second capture): the TP step with every exchange left out -- wrong logits, the
        # per-rank compute time -- so the exchange's share of the step is a measured difference, not count x stand-alone latency
        self.skip_exchange = False
        self._noexch_a = None
        self.device = torch.device(device)
        self.B = batch_size
        self.n_layers = num_layers or shape.num_hidden_layers
        self.tp_rank, self.tp_world, self.tp_group = tp_rank, tp_world, tp_group
        d, Hq, Hkv = shape.head_dim, shape.num_attention_heads, shape.num_key_value_heads
        assert Hkv % tp_world == 0, "KV-head tensor parallelism needs world_size | num_key_value_heads"
        self.Hq_loc, self.Hkv_loc = Hq // tp_world, Hkv // tp_world
        self.d = d

        class _Cfg:
            pass

        cfg = _Cfg()
        cfg.num_hidden_layers = self.n_layers
        cfg.num_key_value_heads = Hkv
        cfg.num_attention_heads = Hq
        cfg.hidden_size = shape.hidden_size
        g = torch.Generator(device=self.device).manual_seed(seed)
        hash_func = torch.randn((d, K * L), generator=g, device=self.device, dtype=torch.float32).to(torch.bfloat16)
        self.server = LSHSparseAttnServer(cfg, K=K, L=L, batch_size=batch_size, max_length=max_length,
                                          generation_buffer=generation_buffer, dense_layers=dense_layers, device=device,
                                          hash_func=hash_func, num_key_value_heads=self.Hkv_loc,
                                          num_attention_heads=self.Hq_loc, max_query_tokens=max_query_tokens,
                                          num_contexts=num_contexts, dense_tail_rows=dense_tail_rows, shared_spill=shared_spill,
                                          max_chunk_tokens=max_chunk_tokens)
        self.max_chunk_tokens = max_chunk_tokens
        self.generation_buffer = generation_buffer

        def w(*shape_):
            return (torch.randn(shape_, generator=g, device=self.device, dtype=torch.float32) * 0.02).to(torch.bfloat16)

        hs, it = shape.hidden_size, shape.intermediate_size
        sl = tp.megatron_slices(Hq, Hkv, d, it, tp_rank, tp_world)
        mega = tp_world > 1 and tp_mode == "megatron"
        self.it_loc = (it // tp_world) if mega else it
        self.layers = []
        for _ in range(self.n_layers):
            # every rank draws the FULL matrices from the same seed and keeps its slice, so that a TP run and a single-GPU run
            # of the same seed are the same model
            wq, wk, wv = w(Hq * d, hs), w(Hkv * d, hs), w(Hkv * d, hs)
            wo, wgu, wd = w(hs, Hq * d), w(2 * it, hs), w(hs, it)
            lw = dict(
                ln1=torch.ones(hs, device=self.device, dtype=torch.bfloat16),
                # this rank's head slice of the q/k/v projections, fused into one GEMM
                wqkv=torch.cat([wq[sl["q_rows"]], wk[sl["kv_rows"]], wv[sl["kv_rows"]]], dim=0).contiguous(),
                wo=(wo[:, sl["wo_cols"]].contiguous() if mega else wo),
                ln2=torch.ones(hs, device=self.device, dtype=torch.bfloat16),
                # [gate rows; up rows] of this rank's slice of the intermediate dimension
                w_gate_up=(torch.cat([wgu[:it][sl["inter"]], wgu[it:][sl["inter"]]], dim=0).contiguous() if mega else wgu),
                w_down=(wd[:, sl["inter"]].contiguous() if mega else wd),
            )
            del wq, wk, wv, wo, wgu, wd
            self.layers.append(lw)
        self.embed = w(shape.vocab_size, hs)
        self.lm_head = w(shape.vocab_size, hs)
        self.norm = torch.ones(hs, device=self.device, dtype=torch.bfloat16)
        self.cos, self.sin = rope_tables(shape.rope_theta, d, max_length + 8, self.device)
        # static step buffers (CUDA-graph friendly)
        self.ids = torch.zeros((batch_size, 1), dtype=torch.long, device=self.device)
        self.pos = torch.zeros((batch_size,), dtype=torch.long, device=self.device)
        self.logits = torch.zeros((batch_size, shape.vocab_size), dtype=torch.float32, device=self.device)
        # step_tokens: the T candidate tokens of each request and the logits after each of them
        self.max_query_tokens = max_query_tokens
        if max_query_tokens > 1:
            self.ids_tok = torch.zeros((batch_size, max_query_tokens), dtype=torch.long, device=self.device)
            self.logits_tok = torch.zeros((batch_size, max_query_tokens, shape.vocab_size), dtype=torch.float32, device=self.device)
        self._gather_buf = None
        self.peer = None
        if tp_world > 1:
            self._gather_buf = torch.empty((tp_world, batch_size, self.Hq_loc * d), dtype=torch.bfloat16, device=self.device)
            if tp_transport == "peer":
                from .peer import PeerExchange
                # one exchange object: slots of max(head outputs, hidden) bytes per rank
                self.peer = PeerExchange(self.server.ctx, tp_rank, tp_world, batch_size * max(self.Hq_loc * d * tp_world, hs) * 2, tp_group)
        self.n_collectives = 0
        self.graph = None
        self.aux_launches_per_step = 0
        # sampling state (sample(), capture(sample=True), generate()): per-request parameters and the Philox counter on the device,
        # and the record of generated tokens the sampler appends to (int32 (B, max_length), allocated on first use)
        self.temperature = torch.zeros((batch_size,), dtype=torch.float32, device=self.device)
        self.top_p = torch.ones((batch_size,), dtype=torch.float32, device=self.device)
        self.sample_offset = torch.zeros((1,), dtype=torch.int64, device=self.device)
        self.sample_seed = 0
        self.sample_status = torch.zeros(((batch_size + 31) // 32,), dtype=torch.int32, device=self.device)
        self.gen_tokens = self.gen_count = self.gen_done = None
        self.eos_token_ids = tuple(shape.eos_token_ids)
        self._gen_graph = None
        self._gen_graph_key = None
        # speculative decoding (spec_step(), capture(draft_tokens=k), generate(draft_tokens=k)): the token history (prompt, then
        # generated tokens) the drafts are looked up in and verify_sample appends to, int32 (B, max_length), with device lengths,
        # limits and done flags, and the per-request step / accepted-draft counters; allocated on first use
        self.token_history = self.history_len = self.history_limit = None
        self.spec_steps = self.spec_accepted = None
        self.ngram = (1, 3)
        self._spec_rows = self._spec_drop = None
        self._spec_graph = None
        self._spec_graph_key = None
        self.last_generate_stats = None
        # sampling filters (set_sampling(top_k=.., ..)): per-request device values, the penalty table (allocated on first use) and
        # whether any value is not neutral, which selects the filtered sampling calls
        self.top_k = torch.zeros((batch_size,), dtype=torch.int32, device=self.device)
        self.min_p = torch.zeros((batch_size,), dtype=torch.float32, device=self.device)
        self.repetition_penalty = torch.ones((batch_size,), dtype=torch.float32, device=self.device)
        self.presence_penalty = torch.zeros((batch_size,), dtype=torch.float32, device=self.device)
        self.frequency_penalty = torch.zeros((batch_size,), dtype=torch.float32, device=self.device)
        self.penalty_table = None
        self._filter_host = {k: [v] * batch_size for k, v in FILTER_NEUTRAL.items()}
        self.filters_active = False

    # ------------------------------------------------------------------------------------------
    def synthetic_prefill(self, P: int, seed: int = 100, dist: str = "gauss", shared: bool = False):
        """Fill every layer's cache with a synthetic P-token context through fill()/build_table().  shared=True: every request
        holds the same context -- request 0 is filled and forked to the others when the server has fewer contexts than requests,
        each request is filled with the same tensors otherwise."""
        srv = self.server
        g = torch.Generator(device=self.device).manual_seed(seed + 7919 * self.tp_rank)
        Hkv, d = self.Hkv_loc, self.d
        fork = shared and srv.ctx.num_contexts < self.B
        for b in range(1 if shared else self.B):
            srv.alloc_buffer(P)
            for layer in range(self.n_layers):
                k = torch.randn((P, Hkv, d), generator=g, device=self.device, dtype=torch.float32)
                if dist == "clustered":
                    nc = 8
                    centres = torch.randn((nc, Hkv, d), generator=g, device=self.device)
                    assign = torch.randint(0, nc, (P,), generator=g, device=self.device)
                    k = k + torch.rand((P, 1, 1), generator=g, device=self.device) * 1.5 * centres[assign]
                k = k.to(torch.bfloat16)
                v = torch.randn((P, Hkv, d), generator=g, device=self.device, dtype=torch.float32).to(torch.bfloat16)
                for r in ([b] if fork or not shared else range(self.B)):
                    srv.fill(layer, r, k, v, P)
                    srv.build_table(layer, r, P)
                del k, v
        if fork:
            srv.fork(0, range(1, self.B))
        self.pos.fill_(P - 1)
        torch.cuda.synchronize(self.device)

    def prefill(self, ids: torch.Tensor, request: int = 0, chunk_size: int = 8192):
        """The reference's LLM.prefill (llama.py:304-325) for one request: ids (P,) or (1, P) token ids.  Layer by layer, chunk by
        chunk: RMSNorm, the q/k/v projection, RoPE at positions 0 .. P-1, the chunk's K/V into one (P, Hkv, d) cache, the server's
        prefill_attention over cache[:end], wo and the residual; then the MLP of every chunk; then fill() and build_table() of the
        layer.  Afterwards self.pos[request] = P - 1 and self.logits[request] holds the logits after the last prompt token: the state
        synthetic_prefill leaves, so a captured step() continues the generation.  With fewer contexts than requests the prompt goes
        into request 0 and every other request is forked from it (as synthetic_prefill(shared=True)).  Prompts of P <= num_sink +
        num_local or P > max_length are refused before anything is written.  Eager library GEMMs; synchronises, not capturable."""
        assert self.tp_world == 1, "prefill is built for a single GPU"
        sh, srv = self.shape, self.server
        ids = ids.to(self.device).long().reshape(-1)
        P = ids.numel()
        chunks = plan_prefill_chunks(P, chunk_size, srv.num_sink_tokens, srv.num_local_tokens, srv.max_length)
        fork = srv.ctx.num_contexts < self.B
        if fork and request != 0:
            raise ValueError(f"with {srv.ctx.num_contexts} contexts for {self.B} requests the prompt goes into request 0 (got {request})")
        if not 0 <= request < self.B:
            raise ValueError(f"request {request} outside [0, {self.B})")
        d, Hq, Hkv, hs, it = self.d, self.Hq_loc, self.Hkv_loc, sh.hidden_size, self.it_loc
        srv.alloc_buffer(P)
        k_cache = torch.empty((P, Hkv, d), dtype=torch.bfloat16, device=self.device)
        v_cache = torch.empty_like(k_cache)
        h = F.embedding(ids, self.embed)   # (P, hs)
        cos, sin = self.cos[:P, None, :], self.sin[:P, None, :]

        def rope(x, a, b):   # x (n, H, d) at positions a .. b-1, rotate-half (models/utils.py:36-44)
            x1, x2 = x[..., : d // 2], x[..., d // 2:]
            return x * cos[a:b] + torch.cat([-x2, x1], dim=-1) * sin[a:b]

        for li, lw in enumerate(self.layers):
            for a, b in chunks:
                x = F.rms_norm(h[a:b], (hs,), lw["ln1"], sh.rms_norm_eps)
                qkv = F.linear(x, lw["wqkv"])   # (n, (Hq+2Hkv)d)
                n = b - a
                q = rope(qkv[:, : Hq * d].reshape(n, Hq, d), a, b)
                k_cache[a:b] = rope(qkv[:, Hq * d:(Hq + Hkv) * d].reshape(n, Hkv, d), a, b)
                v_cache[a:b] = qkv[:, (Hq + Hkv) * d:].reshape(n, Hkv, d)
                o = srv.prefill_attention(q, k_cache[:b], v_cache[:b], causal=True, kv_layout="NHD")
                h[a:b] += F.linear(o.reshape(n, Hq * d), lw["wo"])
            for a, b in chunks:
                x = F.rms_norm(h[a:b], (hs,), lw["ln2"], sh.rms_norm_eps)
                gu = F.linear(x, lw["w_gate_up"])
                h[a:b] += F.linear(F.silu(gu[:, :it]) * gu[:, it:], lw["w_down"])
            srv.fill(li, request, k_cache, v_cache, P)
            srv.build_table(li, request, P)
        x = F.rms_norm(h[P - 1:], (hs,), self.norm, sh.rms_norm_eps)
        self.logits[request] = F.linear(x, self.lm_head).float()[0]
        self.pos[request] = P - 1
        if fork:
            srv.fork(0, range(1, self.B))
            self.pos.fill_(P - 1)
            self.logits[1:] = self.logits[0]
        torch.cuda.synchronize(self.device)
        return self.logits[request]

    def fork(self, src: int, dst: int):
        """Request dst continues from request src: the server's fork (shared context, copied window and dense KV) and src's
        position."""
        self.server.fork(src, dst)
        self.pos[dst] = self.pos[src]

    def reorder(self, src_of: torch.Tensor):
        """Request b continues request src_of[b]: the server's reorder (device int32 (B,), sources are fixed points) and the
        sources' positions.  Capturable."""
        assert self.tp_world == 1, "reorder is built for a single GPU"
        self.server.reorder(src_of)
        self.pos.copy_(self.pos.index_select(0, src_of.long()))

    def beam_select(self, scores: torch.Tensor):
        """The choice of one beam-search step from self.logits (after step()): scores (B,) fp32 are the beams' log-probabilities.
        Returns (parents, tokens, new_scores), each (B,): new beam i extends beam parents[i] by tokens[i], with log-probability
        new_scores[i] = scores[parents[i]] + log_softmax(logits[parents[i]])[tokens[i]], the B best of the B * vocab candidates."""
        V = self.logits.shape[1]
        cand = torch.log_softmax(self.logits, dim=-1) + scores[:, None]
        new_scores, flat = cand.reshape(-1).topk(self.B)
        return flat // V, flat % V, new_scores

    def beam_step(self, scores: torch.Tensor):
        """One beam-search step after step(), all on the device (capturable; capture(beam_scores=scores) puts step() and this into
        one graph): beam_select, then the new beams move into their requests (beam_sources + reorder), self.ids[request_of[i]] =
        tokens[i] and scores[request_of[i]] = new_scores[i] in place.  From one prompt held by every request, start with scores
        [0, -inf, ...]: the B beams then start from distinct tokens of beam 0.  Returns (parents, tokens, request_of)."""
        assert self.tp_world == 1, "beam search is built for a single GPU"
        parents, tokens, new_scores = self.beam_select(scores)
        src_of, request_of = beam_sources(parents)
        self.reorder(src_of)
        req = request_of.long()
        self.ids[req, 0] = tokens
        scores[req] = new_scores
        return parents, tokens, request_of

    # ------------------------------------------------------------------------------------------
    def set_sampling(self, temperature=None, top_p=None, seed: int | None = None, offset: int | None = None, *, top_k=None, min_p=None,
                     repetition_penalty=None, presence_penalty=None, frequency_penalty=None):
        """Per-request sampling parameters for sample(): temperature / top_p scalars or length-B sequences (a temperature below 0.1
        is greedy, as in the reference's LLM.generate), the Philox seed (a host value a captured graph keeps) and the device
        counter offset.  Not capturable (host -> device copies).
        top_k, min_p, repetition_penalty, presence_penalty, frequency_penalty (keyword only; scalars or B values; None keeps the
        current ones): the sampling filters (ops.SampleFilters states them), checked against their ranges (ValueError) before any
        value is written.  While any of them is not neutral, sample(), spec_step() and the graphs captured then run the filtered
        calls on self.penalty_table (ops.penalty_table() builds it from prompts; generate() does)."""
        fv = filter_values(self.B, top_k=top_k, min_p=min_p, repetition_penalty=repetition_penalty,
                           presence_penalty=presence_penalty, frequency_penalty=frequency_penalty)
        for name, vals in fv.items():
            buf = getattr(self, name)
            buf.copy_(torch.tensor(vals, dtype=buf.dtype))
            self._filter_host[name] = vals
        self.filters_active = any(v != FILTER_NEUTRAL[k] for k, vals in self._filter_host.items() for v in vals)
        for name, val, buf in (("temperature", temperature, self.temperature), ("top_p", top_p, self.top_p)):
            if val is None:
                continue
            v = per_request(val, self.B, name)
            if name == "temperature":
                v = [0.0 if t < GREEDY_TEMPERATURE else t for t in v]   # llama.py:340-343: argmax below 0.1
            buf.copy_(torch.tensor(v, dtype=torch.float32))
        if seed is not None:
            self.sample_seed = int(seed)
        if offset is not None:
            self.sample_offset.fill_(int(offset))

    def _penalty_table(self) -> torch.Tensor:
        if self.penalty_table is None:
            self.penalty_table = torch.zeros((self.B, self.shape.vocab_size), dtype=torch.int32, device=self.device)
        return self.penalty_table

    def sample_filters(self):
        """The ops.SampleFilters of the runner's device values and penalty table while a filter is set, else None."""
        if not self.filters_active:
            return None
        return ops.SampleFilters(self.top_k, self.min_p, self.repetition_penalty, self.presence_penalty, self.frequency_penalty,
                                 self._penalty_table())

    def _gen_record(self):
        if self.gen_tokens is None:
            M = self.server.max_length
            self.gen_tokens = torch.zeros((self.B, M), dtype=torch.int32, device=self.device)
            self.gen_count = torch.zeros((self.B,), dtype=torch.int32, device=self.device)
            self.gen_done = torch.zeros((self.B,), dtype=torch.int32, device=self.device)
        return self.gen_tokens, self.gen_count, self.gen_done

    def _history(self):
        if self.token_history is None:
            B, M = self.B, self.server.max_length
            z = lambda *shape: torch.zeros(shape, dtype=torch.int32, device=self.device)  # noqa: E731
            self.token_history = z(B, M)
            self.history_len, self.history_limit = z(B), z(B)
            self.spec_steps, self.spec_accepted = z(B), z(B)
            self._spec_rows, self._spec_drop = z(B * ops.MAX_VERIFY_TOKENS * 2), z(B)
            self._gen_record()
        return self.token_history, self.history_len, self.history_limit, self.gen_done

    def _verify(self, logits: torch.Tensor, count: bool = True):
        """verify_sample of logits (B, T, V) against self.ids_tok into the history, with drop into self._spec_drop."""
        hist, length, limit, done = self._history()
        T = logits.shape[1]
        ops.verify_sample(logits, self.temperature, self.top_p, self.sample_seed, self.sample_offset, self.ids_tok,
                          rows=self._spec_rows[:self.B * T * 2].view(self.B, T, 2), drop=self._spec_drop, history=hist, length=length,
                          limit=limit, done=done, steps=self.spec_steps if count else None,
                          accepted=self.spec_accepted if count else None, eos_token_ids=self.eos_token_ids, status=self.sample_status,
                          filters=self.sample_filters())

    def spec_step(self, T: int, draft: str | None = "ngram"):
        """One step of speculative decoding, all on the device (capturable; capture(draft_tokens=T - 1) puts it into one graph).
        self.ids_tok[:, 0] holds each request's last emitted token.  draft="ngram": prompt-lookup drafts from self.token_history
        (ops.ngram_draft with self.ngram = (g_min, g_max)) into self.ids_tok[:, 1:T]; draft=None: the caller's drafts already there.
        Then step_tokens(T), verify_sample (the accepted drafts and one final token are appended to the history, the final token goes
        to self.ids_tok[:, 0]), server.rewind(drop), self.pos -= drop, self.sample_offset += 1.  Each request advances by its
        accepted drafts + 1; a request whose done flag is set rewinds its whole step."""
        assert self.tp_world == 1, "speculative decoding is built for a single GPU"
        assert 1 <= T <= self.max_query_tokens, f"T={T} outside [1, max_query_tokens={self.max_query_tokens}]"
        hist, length, _, _ = self._history()
        if draft == "ngram":
            ops.ngram_draft(hist, length, self.ids_tok, T, *self.ngram)
        elif draft is not None:
            raise ValueError(f"draft must be 'ngram' or None, got {draft!r}")
        self.step_tokens(T)
        self._verify(self.logits_tok[:, :T])
        self.server.rewind(self._spec_drop)
        self.pos.sub_(self._spec_drop.long())
        self.sample_offset.add_(1)
        return self.ids_tok

    def sample(self, temperature=None, top_p=None):
        """The next token of every request from self.logits into self.ids[:, 0], on the device (one mpig_aux_sample launch: the
        rule is stated in include/magicpig_b200_aux.h), then self.sample_offset += 1.  The token is also appended to the request's
        record (gen_tokens / gen_count) unless gen_done is set; gen_done is set at an id of self.eos_token_ids.  temperature /
        top_p: None keeps the device values (set_sampling()); given, they are written first (not capturable then).  Capturable
        with None; capture(sample=True) puts step() and this into one graph."""
        assert self.tp_world == 1, "sampling is built for a single GPU"
        if temperature is not None or top_p is not None:
            self.set_sampling(temperature, top_p)
        tokens, count, done = self._gen_record()
        ops.sample(self.logits, self.temperature, self.top_p, self.sample_seed, self.sample_offset, ids_out=self.ids,
                   tokens_out=tokens, count=count, done=done, eos_token_ids=self.eos_token_ids, status=self.sample_status,
                   filters=self.sample_filters())
        self.sample_offset.add_(1)
        return self.ids

    def generate(self, prompt, max_new_tokens: int, temperature=0.6, top_p=0.9, eos_token_ids=None, seed: int = 0,
                 chunk_size: int = 8192, check_every: int = 16, draft_tokens: int = 0, ngram=(1, 3), top_k=0, min_p=0.0,
                 repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0):
        """The reference's LLM.generate (llama.py:328-360) for the batch.  prompt: one (P,) tensor of token ids for every request
        (prefilled once and forked when the batch has fewer contexts than requests, prefilled into each request otherwise), or a
        list of B prompts, one per request (needs one context per request; lengths may differ).  temperature / top_p: scalars or
        per-request sequences; temperature < 0.1 is greedy (the first argmax), as in the reference.  eos_token_ids (at most 8; None
        = the shape's) end a request, which keeps its EOS token.  Every request gets at most max_new_tokens tokens.
        Order: the sampling graph (step() then sample()) is captured once per runner and seed on a short synthetic context, which is
        then cleared; the prompts are prefilled; the prefill's logits are sampled eagerly; then the graph is replayed, with
        spill_window() whenever the windows are full, and the requests' done flags are read every check_every replays.
        Refused before anything is written: P + max_new_tokens > max_length, prompts the prefill refuses, a generation that needs
        spills the server cannot do.  Returns B host lists of ints.  Single GPU; the runner's state stays as the generation
        leaves it.
        draft_tokens = k >= 1: speculative decoding with k prompt-lookup drafts per step (ngram = (g_min, g_max), see
        ops.ngram_draft), lossless: every token follows the same nucleus distribution as without drafts (not the same draws).  The
        spec_step(k + 1) graph is captured once per (seed, EOS ids, k, ngram) on a short synthetic context, then cleared; the prompts
        are prefilled and written into self.token_history; the first token comes from the prefill's logits through verify_sample
        at T = 1 (which equals sample()); then the graph is replayed at most max_new_tokens - 1 times, with spill_window() every
        spec_spill_every(generation_buffer, k) replays and the done flags read every check_every replays.  Also refused: k + 1 >
        max_query_tokens or > generation_buffer, P + max_new_tokens + k > max_length, a dense tail too short, spills the server cannot
        do (sharing a context without shared_spill, more than spec_spill_every(generation_buffer, k) replays), a bad ngram.  With
        drafts accepted, requests may finish well before max_new_tokens - 1 replays; the replays until the next done read (at most
        check_every - 1) change nothing but cost a step each, so a smaller check_every trades host reads for fewer idle steps.
        self.last_generate_stats then holds the per-request steps, accepted drafts and tokens per step.
        top_k, min_p, repetition_penalty, presence_penalty, frequency_penalty: scalars or per-request sequences, the sampling filters
        of set_sampling() (Hugging Face's and vLLM's names and conventions; refused outside their ranges before anything is
        written).  With any of them set, self.penalty_table is built from the prompts before the first token and the graphs run
        the filtered calls, with and without drafts (lossless: every token follows the filtered distribution given its prefix).
        With all of them neutral, generate() runs the unfiltered graph and returns what it returns without them."""
        assert self.tp_world == 1, "generate is built for a single GPU"
        srv, B = self.server, self.B
        prompts, shared = generate_prompts(prompt, B, srv.ctx.num_contexts)
        eos = tuple(int(e) for e in (self.shape.eos_token_ids if eos_token_ids is None else eos_token_ids))
        lengths = [int(p.numel()) for p in prompts]
        can_spill = srv.ctx.num_contexts == B or srv.ctx.shared_spill
        filters = dict(top_k=top_k, min_p=min_p, repetition_penalty=repetition_penalty, presence_penalty=presence_penalty,
                       frequency_penalty=frequency_penalty)
        check_generate_args(lengths, max_new_tokens, check_every, eos, srv.max_length,
                            srv.num_sink_tokens, srv.num_local_tokens, chunk_size, self.generation_buffer, can_spill=can_spill,
                            B=B, filters=filters)
        if filter_values(B, **filters) != {k: [v] * B for k, v in FILTER_NEUTRAL.items()}:   # the table will mark the prompts' ids
            for p in prompts:
                if p.numel() and (int(p.min()) < 0 or int(p.max()) >= self.shape.vocab_size):
                    raise ValueError(f"prompt: token ids must lie in [0, {self.shape.vocab_size})")
        if draft_tokens:
            check_spec_args(lengths, max_new_tokens, draft_tokens, ngram, self.max_query_tokens, self.generation_buffer,
                            srv.max_length, srv.ctx.dense_tail_rows if srv.dense_layers else 0, can_spill)
            self.set_sampling(**filters)
            return self._generate_spec(prompts, shared, max_new_tokens, temperature, top_p, eos, seed, chunk_size, check_every,
                                       int(draft_tokens), tuple(int(g) for g in ngram))
        temps = per_request(temperature, B, "temperature")
        tops = per_request(top_p, B, "top_p")
        self.eos_token_ids = eos
        self.set_sampling(**filters)
        key = (int(seed), eos, self.filters_active)
        if self._gen_graph is None or self._gen_graph_key != key:
            # the capture's warm-up steps advance the state: capture on a short synthetic context, then clear it
            self.sample_seed = int(seed)
            self._gen_graph = None
            srv.clear()
            self.synthetic_prefill(srv.num_sink_tokens + srv.num_local_tokens + 64, shared=srv.ctx.num_contexts < B)
            prev = self.graph
            self.capture(sample=True)
            self._gen_graph, self.graph = self.graph, prev
            self._gen_graph_key = key
        self._prefill_prompts(prompts, shared, chunk_size)
        if self.filters_active:
            ops.penalty_table(prompts, self.shape.vocab_size, out=self._penalty_table())
        tokens, count, done = self._gen_record()
        count.zero_()
        done.zero_()
        self.sample_status.zero_()
        self.set_sampling(temps, tops, seed=seed, offset=0)
        self.sample()   # the first token, from the prefill's logits
        used = 0        # generated rows in the windows
        for i in range(max_new_tokens - 1):
            if i % check_every == 0 and bool(done.all()):
                break
            if used == self.generation_buffer:
                srv.spill_window()
                used = 0
            self._gen_graph.replay()
            used += 1
        n = count.tolist()
        if int(self.sample_status.any()):
            raise N.MagicPigError("generate: a request's logits held NaN / +inf or no finite value (its token was set to 0)")
        rows = tokens[:, :max(n)].tolist() if max(n) else [[] for _ in range(B)]
        return [rows[b][:n[b]] for b in range(B)]

    def _prefill_prompts(self, prompts, shared: bool, chunk_size: int):
        srv = self.server
        srv.clear()
        if shared and srv.ctx.num_contexts < self.B:
            self.prefill(prompts[0], chunk_size=chunk_size)
        else:
            for b, p in enumerate(prompts):
                self.prefill(p, request=b, chunk_size=chunk_size)

    def _generate_spec(self, prompts, shared, max_new_tokens, temperature, top_p, eos, seed, chunk_size, check_every, k, ngram):
        """generate(draft_tokens=k) after its checks (see generate())."""
        srv, B, T = self.server, self.B, k + 1
        temps = per_request(temperature, B, "temperature")
        tops = per_request(top_p, B, "top_p")
        self.eos_token_ids = eos
        hist, length, limit, done = self._history()
        key = (int(seed), eos, k, ngram, self.filters_active)
        if self._spec_graph is None or self._spec_graph_key != key:
            # the capture's warm-up steps advance the state: capture on a short synthetic context, then clear it
            self.sample_seed, self.ngram = int(seed), ngram
            self._spec_graph = None
            srv.clear()
            self.synthetic_prefill(srv.num_sink_tokens + srv.num_local_tokens + 64, shared=srv.ctx.num_contexts < B)
            length.zero_()
            limit.fill_(hist.shape[1])
            done.zero_()
            prev = self.graph
            self.capture(warm=max(1, min(3, self.generation_buffer // T - 1)), draft_tokens=k)
            self._spec_graph, self.graph = self.graph, prev
            self._spec_graph_key = key
        self._prefill_prompts(prompts, shared, chunk_size)
        if self.filters_active:
            ops.penalty_table(prompts, self.shape.vocab_size, out=self._penalty_table())
        P = [int(p.numel()) for p in prompts]
        for b, p in enumerate(prompts):
            hist[b, :P[b]] = p.to(self.device, torch.int32)
        length.copy_(torch.tensor(P, dtype=torch.int32))
        limit.copy_(torch.tensor([n + int(max_new_tokens) for n in P], dtype=torch.int32))
        done.zero_()
        self.spec_steps.zero_()
        self.spec_accepted.zero_()
        self.sample_status.zero_()
        self.set_sampling(temps, tops, seed=seed, offset=0)
        self._verify(self.logits[:, None], count=False)   # the first token, from the prefill's logits: T = 1 is sample()
        self.sample_offset.add_(1)
        every = spec_spill_every(self.generation_buffer, k)
        since = 0   # replays since the last spill
        for i in range(max_new_tokens - 1):
            if i % check_every == 0 and bool(done.all()):
                break
            if since == every:
                srv.spill_window()
                since = 0
            self._spec_graph.replay()
            since += 1
        n = length.tolist()
        if int(self.sample_status.any()):
            raise N.MagicPigError("generate: a request's logits held NaN / +inf or no finite value (its token was set to 0)")
        steps, acc = self.spec_steps.tolist(), self.spec_accepted.tolist()
        self.last_generate_stats = dict(draft_tokens=k, steps=steps, accepted=acc, tokens=[n[b] - P[b] for b in range(B)],
                                        tokens_per_step=(sum(n) - sum(P) - B) / max(sum(steps), 1))
        return [hist[b, P[b]:n[b]].tolist() for b in range(B)]

    # ------------------------------------------------------------------------------------------
    def _rope(self, x: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
        # x (B, H, 1, d); rotate-half convention (models/utils.py:36-44)
        cos = self.cos[pos][:, None, None, :]
        sin = self.sin[pos][:, None, None, :]
        x1, x2 = x[..., : self.d // 2], x[..., self.d // 2:]
        return x * cos + torch.cat([-x2, x1], dim=-1) * sin

    def step(self):
        """One decode token for the whole batch: reads self.ids, advances self.pos, writes self.logits."""
        return self._step_fused() if self.fused else self._step_eager()

    def _step_fused(self):
        """Same math as _step_eager with the per-layer elementwise glue in three fused kernels
        (include/magicpig_b200_aux.h): residual-add + RMSNorm, RoPE + q/k/v split, SiLU*up."""
        sh, srv = self.shape, self.server
        B, d, Hq, Hkv = self.B, self.d, self.Hq_loc, self.Hkv_loc
        lib = srv.ctx.lib
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
        n_aux = [0]

        def AUX(rc):   # one launch of a harness kernel (include/magicpig_b200_aux.h)
            n_aux[0] += 1
            N.check(rc)

        hs, it = sh.hidden_size, self.it_loc
        mega = self.tp_world > 1 and self.tp_mode == "megatron"
        n_coll = [0]
        self.pos.add_(1)
        srv.plan()
        h = F.embedding(self.ids, self.embed).reshape(B, hs).contiguous()
        x = torch.empty_like(h)
        q = torch.empty((B, Hq, 1, d), dtype=torch.bfloat16, device=self.device)
        k = torch.empty((B, Hkv, 1, d), dtype=torch.bfloat16, device=self.device)
        v = torch.empty((B, Hkv, 1, d), dtype=torch.bfloat16, device=self.device)
        act = torch.empty((B, it), dtype=torch.bfloat16, device=self.device)
        # decode-batch linear layers: weight-streaming GEMV (mpig_aux_gemv) where it applies, library GEMM otherwise
        nqkv = (Hq + 2 * Hkv) * d
        qkv_buf = torch.empty((B, nqkv), dtype=torch.bfloat16, device=self.device)
        o_buf = torch.empty((B, hs), dtype=torch.bfloat16, device=self.device)
        d_buf = torch.empty((B, hs), dtype=torch.bfloat16, device=self.device)

        def linear(inp, wt, out, swiglu=0):
            n_out, k_in = (wt.shape[0] // 2 if swiglu else wt.shape[0]), wt.shape[1]
            if self.use_gemv and B <= self.GEMV_MAX_ROWS and k_in % 256 == 0 and B * k_in * 2 <= 200 * 1024:
                AUX(lib.mpig_aux_gemv(P(wt), P(inp), P(out), B, n_out, k_in, swiglu, st))
                return out
            if swiglu:
                gu = F.linear(inp, wt)
                AUX(lib.mpig_aux_silu_mul(P(gu), P(out), B, n_out, st))
                return out
            return F.linear(inp, wt)

        delta = None
        fuse = self.use_gemv and B <= self.GEMV_MAX_ROWS and hs % 256 == 0 and B * hs * 2 <= 200 * 1024 and d == 128
        h2 = torch.empty_like(h)   # second buffer of the ping-ponged residual stream (fused prologue)
        PN = lambda t: P(t) if t is not None else None  # noqa: E731
        for li, lw in enumerate(self.layers):
            if fuse:
                # residual add + RMSNorm + q/k/v projection + RoPE/split in one weight-streaming kernel
                AUX(lib.mpig_aux_norm_qkv_rope(P(lw["wqkv"]), P(h), PN(delta), P(lw["ln1"]), sh.rms_norm_eps, P(h2), P(self.cos),
                                                   P(self.sin), P(self.pos), P(q), P(k), P(v), B, Hq, Hkv, hs, st))
                h, h2 = h2, h
            else:
                AUX(lib.mpig_aux_add_rmsnorm(P(h), PN(delta), P(lw["ln1"]), sh.rms_norm_eps, P(x), B, hs, st))
                qkv = linear(x, lw["wqkv"], qkv_buf)
                AUX(lib.mpig_aux_rope_split(P(qkv), P(self.cos), P(self.sin), P(self.pos), P(q), P(k), P(v), B, Hq, Hkv, st))
            if self.skip_exchange and self.tp_world > 1 and not self.skip_sparse:
                srv.decode(q, k, v, li)
                if self._noexch_a is None:
                    self._noexch_a = torch.zeros((B, lw["wo"].shape[1]), dtype=torch.bfloat16, device=self.device)
                a = self._noexch_a
            elif self.peer is not None and self.tp_mode == "ag" and li not in srv.dense_layers:
                # head outputs stored straight into every peer's gather buffer by the attention kernel's epilogue
                a = self.peer.decode_allgather(li, q, k, v)
                n_coll[0] += 1
            elif self.skip_sparse and li not in srv.dense_layers:
                a = q.reshape(B, Hq * d)   # measurement aid (MPIG_SKIP_ATTN=1): what the step costs without the hot path
            else:
                a = srv.decode(q, k, v, li).reshape(B, Hq * d)  # <- the hot path
                if self.tp_world > 1 and self.tp_mode == "ag":
                    a = (self.peer.all_gather(a) if self.peer is not None
                         else tp.gather_head_outputs(a, self.tp_world, self.tp_group, self._gather_buf))
                    n_coll[0] += 1
            o = linear(a.contiguous(), lw["wo"], o_buf)
            if mega and not self.skip_exchange:
                o = self.peer.all_reduce(o) if self.peer is not None else tp.all_reduce_sum(o, self.tp_group)
                n_coll[0] += 1
            if fuse:
                # residual add + RMSNorm + gate/up projection + SwiGLU
                AUX(lib.mpig_aux_norm_gemv(P(lw["w_gate_up"]), P(h), P(o), P(lw["ln2"]), sh.rms_norm_eps, P(h2), P(act), B, it, hs, 1, st))
                h, h2 = h2, h
            else:
                AUX(lib.mpig_aux_add_rmsnorm(P(h), P(o), P(lw["ln2"]), sh.rms_norm_eps, P(x), B, hs, st))
                linear(x, lw["w_gate_up"], act, swiglu=1)
            delta = linear(act, lw["w_down"], d_buf)
            if mega and not self.skip_exchange:
                delta = self.peer.all_reduce(delta) if self.peer is not None else tp.all_reduce_sum(delta, self.tp_group)
                n_coll[0] += 1
        AUX(lib.mpig_aux_add_rmsnorm(P(h), P(delta), P(self.norm), sh.rms_norm_eps, P(x), B, hs, st))
        self.logits.copy_(F.linear(x, self.lm_head).float())
        self.aux_launches_per_step = n_aux[0]
        self.n_collectives = n_coll[0]
        return self.logits

    def _step_eager(self):
        sh, srv = self.shape, self.server
        B, d, Hq, Hkv = self.B, self.d, self.Hq_loc, self.Hkv_loc
        self.pos.add_(1)
        srv.plan()
        h = F.embedding(self.ids, self.embed)  # (B,1,hs)
        for li, lw in enumerate(self.layers):
            x = F.rms_norm(h, (sh.hidden_size,), lw["ln1"], sh.rms_norm_eps)
            qkv = F.linear(x, lw["wqkv"])  # (B,1,(Hq+2Hkv)d)
            q = qkv[..., : Hq * d].reshape(B, 1, Hq, d).transpose(1, 2)
            k = qkv[..., Hq * d:(Hq + Hkv) * d].reshape(B, 1, Hkv, d).transpose(1, 2)
            v = qkv[..., (Hq + Hkv) * d:].reshape(B, 1, Hkv, d).transpose(1, 2)
            q = self._rope(q, self.pos)
            k = self._rope(k, self.pos)
            a = srv.decode(q, k, v, li)  # (B,1,Hq_loc*d)   <- the hot path
            mega = self.tp_world > 1 and self.tp_mode == "megatron"
            if self.tp_world > 1 and not mega:
                # KV-head TP: one all-gather of head outputs per layer (north-star), weights replicated
                a = tp.gather_head_outputs(a.reshape(B, Hq * d), self.tp_world, self.tp_group, self._gather_buf)
                a = a.reshape(B, 1, self.tp_world * Hq * d)
            o = F.linear(a, lw["wo"])
            if mega:
                o = tp.all_reduce_sum(o.contiguous(), self.tp_group)
            h = h + o
            x = F.rms_norm(h, (sh.hidden_size,), lw["ln2"], sh.rms_norm_eps)
            gu = F.linear(x, lw["w_gate_up"])
            it = self.it_loc
            dn = F.linear(F.silu(gu[..., :it]) * gu[..., it:], lw["w_down"])
            if mega:
                dn = tp.all_reduce_sum(dn.contiguous(), self.tp_group)
            h = h + dn
        x = F.rms_norm(h[:, -1], (sh.hidden_size,), self.norm, sh.rms_norm_eps)
        self.logits.copy_(F.linear(x, self.lm_head).float())
        return self.logits

    def step_tokens(self, T: int, drop: torch.Tensor | None = None):
        """A verification step of T tokens for the whole batch (speculative decoding): reads the candidates self.ids_tok[:, :T],
        writes self.logits_tok[:, :T] (B, T, vocab), the logits after each candidate, and advances self.pos by T.  Eager-path math
        (library GEMMs over the B*T rows) with per-token RoPE positions pos+1 .. pos+T; the attention server checks the T
        tokens in one pass per layer (plan(T), decode of (B, H, T, d)).  With `drop` (device int32 (B,): rejected tokens per
        request) the step ends with server.rewind(drop) and self.pos falls back by drop.  Graph-capturable; step() is separate."""
        assert self.tp_world == 1, "verification steps are built for a single GPU"
        assert 1 <= T <= self.max_query_tokens, f"T={T} outside [1, max_query_tokens={self.max_query_tokens}]"
        srv = self.server
        srv.plan(T)
        pos = self.pos[:, None] + torch.arange(1, T + 1, device=self.device)   # (B, T)
        self.pos.add_(T)
        self._forward_tokens(T, pos)   # token t attending causally
        if drop is not None:
            srv.rewind(drop)
            self.pos.sub_(drop.long())
        return self.logits_tok[:, :T]

    def step_tree(self, T: int, parents, nodes=None, count=None):
        """A verification step over a token tree of T nodes: reads the candidates self.ids_tok[:, :T] in node order, writes
        self.logits_tok[:, :T] (B, T, vocab), the logits after each node.  parents: device int32 (B, T) or (T,) (every request),
        or a host sequence (parents[b][0] = -1, 0 <= parents[b][t] < t).  Node t sits at RoPE position pos + 1 + depth(t) and
        attends to the context, its ancestors and itself; the depths are computed on the device.  Same eager-path math as
        step_tokens.  With `nodes` / `count` (device int32 (B, T) / (B,), or host values) the step ends with server.accept(nodes,
        count) and self.pos advances by count; without, every node stays in the caches (accept later) and self.pos advances by T.
        Graph-capturable with device tensors."""
        assert self.tp_world == 1, "verification steps are built for a single GPU"
        assert 1 <= T <= self.max_query_tokens, f"T={T} outside [1, max_query_tokens={self.max_query_tokens}]"
        srv, B = self.server, self.B
        if not (isinstance(parents, torch.Tensor) and parents.is_cuda):
            parents = torch.as_tensor(parents, dtype=torch.int32).to(self.device)
        parents = parents.to(torch.int32)
        if parents.dim() == 1:
            parents = parents[None].expand(B, T)
        parents = parents.contiguous()
        srv.plan(T, parents=parents)
        # depth(t) = depth(parent(t)) + 1: T - 1 gathers settle every node of a topologically ordered tree
        par = parents.long().clamp(min=0)
        depth = torch.zeros((B, T), dtype=torch.long, device=self.device)
        for _ in range(T - 1):
            depth = torch.where(parents >= 0, depth.gather(1, par) + 1, 0)
        pos = self.pos[:, None] + 1 + depth   # (B, T)
        self._forward_tokens(T, pos)   # node t attending to its ancestors
        if count is None:
            self.pos.add_(T)
        else:
            srv.accept(nodes, count)
            if isinstance(count, torch.Tensor):
                self.pos.add_(count.to(self.device).long())
            else:
                self.pos.add_(torch.as_tensor(count if not isinstance(count, int) else [count] * B, device=self.device).long())
        return self.logits_tok[:, :T]

    def extend(self, ids: torch.Tensor, lengths=None):
        """Feed a turn of new prompt tokens to every request (a follow-up turn after generating, or a forked request's question):
        ids (B, T_total) device long, lengths (B,) the real tokens per request (default T_total; the rest of a row is padding).  The
        turn goes in chunk steps of at most min(max_chunk_tokens, generation_buffer) tokens, each with exact causal attention over the
        whole conversation, spill_window() before each (the window keeps its newest num_local_tokens rows), rewind() of the padding.
        Token t of request b sits at RoPE position pos[b] + 1 + t.  Afterwards self.pos has advanced by lengths[b] and self.logits[b]
        holds the logits after request b's last real token (unchanged where lengths[b] = 0), and every window has a free row (a last
        chunk that filled it is spilled), so a captured step() continues the generation.  Before anything is planned, the turn is
        checked against the dense capacity: pos[b] + 1 + lengths[b] <= max_length (with dense_tail_rows, also lengths[b] <= R; the
        exact tail capacity, prompt base + R, is checked by each chunk's plan).  Eager-path math (library GEMMs over the B*T rows of
        a chunk); synchronises, not capturable."""
        assert self.tp_world == 1, "extend is built for a single GPU"
        assert self.max_chunk_tokens > 0, "construct the runner with max_chunk_tokens > 0"
        srv, B = self.server, self.B
        ids = ids.to(self.device).long()
        assert ids.dim() == 2 and ids.shape[0] == B, f"ids must be (B={B}, T_total), got {tuple(ids.shape)}"
        n = [ids.shape[1]] * B if lengths is None else [int(x) for x in torch.as_tensor(lengths).reshape(-1).tolist()]
        assert len(n) == B and all(0 <= x <= ids.shape[1] for x in n), f"lengths {n} outside [0, {ids.shape[1]}]"
        # the dense layers hold every token of the conversation: pos[b] + 1 rows before the turn
        rows = [p + 1 + x for p, x in zip(self.pos.tolist(), n)]
        R = srv.ctx.dense_tail_rows
        if srv.dense_layers and (max(rows) > srv.max_length or (R > 0 and max(n) > R)):
            raise N.MagicPigError(f"extend: a turn of {n} tokens does not fit the dense caches ({rows} rows after it, max_length "
                                  f"{srv.max_length}" + (f", dense_tail_rows {R})" if R > 0 else ")"))
        plan = plan_turn_chunks(n, self.max_chunk_tokens, self.generation_buffer)
        for start, T, drop in plan:
            srv.spill_window()
            srv.plan_chunk(T)
            pos = self.pos[:, None] + 1 + torch.arange(T, device=self.device)   # (B, T)
            h = self._forward_rows(F.embedding(ids[:, start:start + T], self.embed), T, pos)
            last = [x - 1 - start for x in n]   # the row of request b's last real token in this chunk, if it is here
            sel = [b for b in range(B) if 0 <= last[b] < T]
            if sel:
                rows = h[sel, [last[b] for b in sel]]   # (len(sel), hs)
                x = F.rms_norm(rows, (self.shape.hidden_size,), self.norm, self.shape.rms_norm_eps)
                self.logits[sel] = F.linear(x, self.lm_head).float()
            kept = torch.tensor([T - x for x in drop], device=self.device, dtype=torch.long)
            if any(drop):
                srv.rewind(drop)
            self.pos.add_(kept)
        if plan and plan[-1][1] >= self.generation_buffer:
            srv.spill_window()   # the last chunk may have filled a window: the next step() needs a free row
        torch.cuda.synchronize(self.device)
        return self.logits

    def _forward_tokens(self, T: int, pos: torch.Tensor):
        """The eager forward of the T rows of a verification step (after its plan): embeddings of self.ids_tok[:, :T] at RoPE
        positions pos (B, T) through every layer into self.logits_tok[:, :T] (B, T, vocab)."""
        sh = self.shape
        h = self._forward_rows(F.embedding(self.ids_tok[:, :T], self.embed), T, pos)
        x = F.rms_norm(h, (sh.hidden_size,), self.norm, sh.rms_norm_eps)
        self.logits_tok[:, :T].copy_(F.linear(x, self.lm_head).float())

    def _forward_rows(self, h: torch.Tensor, T: int, pos: torch.Tensor) -> torch.Tensor:
        """The layers over the T rows of a step (after its plan): h (B, T, hs) embeddings at RoPE positions pos (B, T) -> the final
        residual stream (B, T, hs).  The attention server decodes the step the plan made (verification, tree or chunk step)."""
        sh, srv = self.shape, self.server
        B, d, Hq, Hkv, hs, it = self.B, self.d, self.Hq_loc, self.Hkv_loc, sh.hidden_size, self.it_loc
        for li, lw in enumerate(self.layers):
            x = F.rms_norm(h, (hs,), lw["ln1"], sh.rms_norm_eps)
            qkv = F.linear(x, lw["wqkv"])   # (B, T, (Hq+2Hkv)d)
            q = self._rope_at(qkv[..., : Hq * d].reshape(B, T, Hq, d).transpose(1, 2), pos)
            k = self._rope_at(qkv[..., Hq * d:(Hq + Hkv) * d].reshape(B, T, Hkv, d).transpose(1, 2), pos)
            v = qkv[..., (Hq + Hkv) * d:].reshape(B, T, Hkv, d).transpose(1, 2)
            a = srv.decode(q, k, v, li)   # (B, T, Hq*d)   <- the hot path
            h = h + F.linear(a, lw["wo"])
            x = F.rms_norm(h, (hs,), lw["ln2"], sh.rms_norm_eps)
            gu = F.linear(x, lw["w_gate_up"])
            h = h + F.linear(F.silu(gu[..., :it]) * gu[..., it:], lw["w_down"])
        return h

    def _rope_at(self, x: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
        # x (B, H, T, d), pos (B, T): token t of request b rotated by its own position
        cos = self.cos[pos][:, None]
        sin = self.sin[pos][:, None]
        x1, x2 = x[..., : self.d // 2], x[..., self.d // 2:]
        return x * cos + torch.cat([-x2, x1], dim=-1) * sin

    def capture(self, warm: int = 3, beam_scores: torch.Tensor | None = None, sample: bool = False, draft_tokens: int = 0):
        """Capture step() into a CUDA graph (launch-bound otherwise: ~600 small kernels per token).  With beam_scores (a device
        fp32 (B,) tensor that stays in place) the graph is step() followed by beam_step(beam_scores); the warm-up steps run it too,
        so reset the beams' state (clear and prefill) before the first replay.  With sample=True the graph is step() followed by
        sample(): each replay writes the next token into self.ids, appends it to the record and advances the Philox offset, with
        the parameters on the device at replay time and the seed at capture time; the warm-up steps sample too.  With
        draft_tokens = k >= 1 the graph is spec_step(k + 1) (prompt-lookup drafts with self.ngram) instead of step(); the warm-up
        steps run it too.  While a sampling filter is set (set_sampling()), the graph's sampling runs the filtered calls on the
        device values and table it finds at replay time."""
        def body():
            if draft_tokens:
                self.spec_step(draft_tokens + 1)
                return
            self.step()
            if beam_scores is not None:
                self.beam_step(beam_scores)
            if sample:
                self.sample()

        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(warm):
                body()
        torch.cuda.current_stream(self.device).wait_stream(s)
        torch.cuda.synchronize(self.device)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            body()
        return warm + 1  # decode steps consumed (window slots used)

    def replay(self):
        self.graph.replay()
        return self.logits
