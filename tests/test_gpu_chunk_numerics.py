"""Chunk steps (attend_chunk_kernel) against fp64 at the shapes the chunk line measures (`-m gpu`).

tests/test_gpu_chunk.py checks chunk steps over ~1 300 store keys with Llama-3.1-8B heads.  Here:

  * (a) the measured shapes: Hq 32, Hkv 8, a 98 000-token prompt (97 932 store keys + 68 window rows), M = P + 2048,
    generation_buffer 1100, B = 1 at T = 64, 256, 1024 and B = 8 on one slot with shared spill at T = 64, 256, each request with
    spilled keys of its own; a 132-SM H100 takes 16 / 4 / 1 / 2 key splits for B1 T64 / B1 T256 / B1 T1024 / B8 T64 (pinned);
  * (b) group sizes 1, 7, 8 and 8 with one kv-head, T = 1, 37, 293, over 20 000 store keys;
  * (c) split edges: an m-block whose last split is empty, one split, store lengths 64k - 1, 64k, 64k + 1, an empty store, a split
    boundary inside the chunk's own rows;
  * (d) a captured plan_chunk -> sparse -> dense replayed, then replayed after an eager spill and after a rewind: the replay reads
    the lengths of the replay, with a split count the host estimated at capture (different from the eager one);
  * (e) eight chunk_attend launches back to back over the shared split scratch and merge tickets.

Every row (request, token, q-head) of fp32 output is held to max|out - o| <= 1e-3 max|o| of an fp64 restatement (IEEE fp64 torch
arithmetic on the same device, none of the library's kernels), the bf16 output must be the fp32 output rounded half-up, and every
case reports its split count (mpig_get_info("chunk_splits")), which must equal the host formula of launch_chunk_attend.

Regimes: R1 key mean (the chunk's keys carry mu; the sparse layer centres them), R2 sinks (the first rows of the window or the
dense cache aligned with every query, a tile at a split boundary carrying a share of the mass too), R4 large logits (queries x 16;
one dominant key at the first key of a split, at the last key of the split before, or as the chunk's own row of token 0).  Before
any library call each case checks that every named perturbation of the restatement (PERTURBATIONS) moves some row by >= 10x the
bar, so that a kernel making that mistake fails.  tests/test_chunk_numerics_inputs_cpu.py runs the generator, restatement and
those checks at a reduced size without a GPU.
"""
import math

import pytest
import torch

from tests.support.chunk_cases import CK_KT, GEN_C, K_, L_, N_C, NL, NS, P_C, Case, d, host_splits, split_per
from tests.support.fp64 import BAR, assert_rounded_half_up, rel_rows
from tests.support.library import DEV, skip_unless_132_sms, two_layer_context


# ------------------------------------------------------------------------------------------------
# GPU side
# ------------------------------------------------------------------------------------------------
def make_ctx(c, M, gen=GEN_C, t_max=1024):
    """A context over case c: layer 0 dense, layer 1 sparse."""
    from magicpig_b200 import synth
    ctx = two_layer_context(K_, L_, c.Hq, c.Hkv, c.B, M, gen, synth.make_hash_func(d, K_, L_, seed=1), dict(out_f32=1),
                            alloc_dense_kv=True, num_contexts=0 if c.C == c.B else c.C,
                            dense_tail_rows=(c.T + 64 if c.tail else 0), shared_spill=c.spill)
    ctx.reserve_chunk_tokens(t_max)
    return ctx


def fill(ctx, c, pre):
    """Fill the context from the case's state `pre` (the store, windows and dense rows before the library's own spill)."""
    for s in range(c.C):
        k, v = pre["store_k"][s], pre["store_v"][s]
        if k.shape[1]:
            ctx.attn_fill(1, s, k.contiguous(), v.contiguous(), k.float().norm(dim=-1).contiguous())
            ctx.lsh_build(1, s, ctx.hash_keys(k.contiguous()))
        ctx.dense_fill(0, s, pre["dk"][s].contiguous(), pre["dv"][s].contiguous(), pre["dk"][s].shape[0])
    for b in range(c.C, c.B):
        ctx.fork(c.slot(b), b)
        if not c.tail:
            ctx.dense_fill(0, b, pre["dk"][b].contiguous(), pre["dv"][b].contiguous(), pre["dk"][b].shape[0])
    for b in range(c.B):
        ctx.window_fill(1, b, c.avg[c.slot(b)].contiguous(), pre["win_k"][b].contiguous(), pre["win_v"][b].contiguous())


def snapshot(c):
    return dict(store_k=[t.clone() for t in c.store_k], store_v=[t.clone() for t in c.store_v], dk=[t.clone() for t in c.dk],
                dv=[t.clone() for t in c.dv], win_k=[t.clone() for t in c.win_k], win_v=[t.clone() for t in c.win_v])


def check_out(c, out, f32, o, label):
    """Per row: max|out_f32 - o| <= BAR max|o|; the bf16 output is the fp32 output rounded half-up.  Returns the worst row."""
    worst = rel_rows(f32, o)
    print(f"{label}: largest relative row error {worst:.2e} ({worst / BAR:.1%} of the bar)")
    assert worst <= BAR, f"{label}: fp32 output differs from fp64 by {worst:.3e} relative (bar {BAR:g})"
    assert_rounded_half_up(out, f32, label)
    return worst


def run_chunk(ctx, c, layers=("sparse", "dense")):
    """plan_chunk(T), then the case's layers; -> {layer: (bf16 out, fp32 out, splits)}."""
    T = c.T
    ctx.plan_chunk(T)
    r = {}
    for layer in layers:
        out = ctx.chunk_attend(1 if layer == "sparse" else 0, T, c.q, c.k, c.v)
        r[layer] = (out.reshape(c.B, T, c.Hq, d), ctx.last_out_f32().reshape(c.B, T, c.Hq, d), ctx.get_info("chunk_splits"))
    return r


def run_case(c, label, M, gen=GEN_C, t_max=1024, pre_spill=None):
    """Self-check the inputs, run one chunk step on both layers and check it against fp64."""
    refs = {}
    for layer in c.layers:
        refs[layer], moved = c.check_inputs(layer)
        print(f"{label} {layer}: " + ", ".join(f"{k} {v:.2e}" for k, v in moved.items()))
    ctx = make_ctx(c, M, gen, t_max)
    fill(ctx, c, pre_spill or snapshot(c))
    if c.spill:
        assert ctx.spill_window().tolist() == c.x
    r = run_chunk(ctx, c, c.layers)
    worst = 0.0
    for layer in c.layers:
        out, f32, sp = r[layer]
        assert sp == c.splits(layer), f"{label} {layer}: chunk_splits {sp}, host formula {c.splits(layer)}"
        worst = max(worst, check_out(c, out, f32, refs[layer], f"{label} {layer} ({sp} splits)"))
    assert ctx.error_flags() == 0
    return worst, r


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def build(regime, B, T, **kw):
    """Case with the spill applied to the case's state; returns (case, the state the context is filled with)."""
    if "sms" not in kw:
        kw["sms"] = sms()
    c = Case(regime, B, T, **kw)
    pre = snapshot(c)
    if not kw.get("spill", False):
        return c, pre
    # the spill rewrote the windows: fill the context with the windows and store as they were, then spill through the library
    for b in range(B):
        s = c.slot(b)
        pre["win_k"][b] = torch.cat([c.win_k[b][:, :NS], *[c.store_k[s][:, lo:hi] for r, lo, hi in c.priv[s] if r == b],
                                     c.win_k[b][:, NS:]], 1)
        pre["win_v"][b] = torch.cat([c.win_v[b][:, :NS], *[c.store_v[s][:, lo:hi] for r, lo, hi in c.priv[s] if r == b],
                                     c.win_v[b][:, NS:]], 1)
    for s in range(c.C):
        pre["store_k"][s], pre["store_v"][s] = pre["store_k"][s][:, :c.stale_n[s]], pre["store_v"][s][:, :c.stale_n[s]]
    return c, pre


# ---- (a) the measured shapes -------------------------------------------------------------------------------------------------
SPILL_X = (40, 67, 101, 133, 170, 199, 230, 255)
MEASURED = [   # (B, T, regime, place)
    (1, 64, "R1", None), (1, 64, "R2", None), (1, 64, "R4", "split_start"),
    (1, 256, "R4", "split_end"),
    (1, 1024, "R1", None), (1, 1024, "R2", None), (1, 1024, "R4", "own_row"),
    (8, 64, "R2", None), (8, 256, "R1", None),
]
PINNED = {(1, 64): (2, 16), (1, 256): (8, 4), (1, 1024): (32, 1), (8, 64): (2, 2)}


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,regime,place", MEASURED, ids=[f"B{b}-T{t}-{r}{'-' + p if p else ''}" for b, t, r, p in MEASURED])
def test_measured_shapes(cuda_lib, B, T, regime, place):
    kw = dict(spill=True, C=1, x=SPILL_X) if B > 1 else {}
    c, pre = build(regime, B, T, place=place or "split_start", seed=100 * B + T + ord(regime[1]), **kw)
    run_case(c, f"B{B} T{T} {regime}", M=P_C + 2048, pre_spill=pre)


@pytest.mark.gpu
@pytest.mark.parametrize("B,T", list(PINNED), ids=[f"B{b}-T{t}" for b, t in PINNED])
def test_measured_shapes_splits(cuda_lib, B, T):
    """The (m-blocks, splits) of the chunk line's shapes on a 132-SM H100, through chunk_splits."""
    skip_unless_132_sms()
    from magicpig_b200.ops import Context
    ctx = Context(K_, L_, 2, 32, 8, d, B, P_C + 2048, NS, NL, GEN_C, dense_layers=[0], alloc_dense_kv=True, device=DEV,
                  num_contexts=1 if B > 1 else 0, shared_spill=B > 1)
    ctx.reserve_chunk_tokens(T)
    z = torch.zeros((8, N_C, d), dtype=torch.bfloat16, device=DEV)
    ctx.attn_fill(1, 0, z, z, z[..., 0].float())
    ctx.dense_fill(0, 0, z[0, :1].expand(P_C, 8, d).contiguous(), z[0, :1].expand(P_C, 8, d).contiguous(), P_C)
    for b in range(1, B):
        ctx.fork(0, b)
    w = torch.zeros((8, NS + NL, d), dtype=torch.bfloat16, device=DEV)
    for b in range(B):
        ctx.window_fill(1, b, w[:, 0].contiguous(), w, w)
    q = torch.zeros((B, T, 32, d), dtype=torch.bfloat16, device=DEV)
    kv = torch.zeros((B, T, 8, d), dtype=torch.bfloat16, device=DEV)
    assert ctx.get_info("chunk_splits") == 0
    ctx.plan_chunk(T)
    got = []
    for layer in (1, 0):
        ctx.chunk_attend(layer, T, q, kv, kv)
        got.append(ctx.get_info("chunk_splits"))
    nmb, want = PINNED[(B, T)]
    assert host_splits(T, 4, 8, B, 132, N_C + NS + NL + T) == (nmb, want)
    assert got == [want, want], f"B={B} T={T}: chunk_splits {got}, want {want}"


# ---- (b) group sizes ---------------------------------------------------------------------------------------------------------
GROUPS = [(8, 8), (28, 4), (64, 8), (8, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 37, 293])
@pytest.mark.parametrize("Hq,Hkv", GROUPS, ids=[f"G{q // k}-Hkv{k}" for q, k in GROUPS])
def test_group_sizes(cuda_lib, Hq, Hkv, T):
    """G = 1, 7 (a token's rows straddle warps and m-blocks), 8 and 8 with one kv-head, over ~20 000 store keys; the dense
    layer in shared-prefix mode for G = 7 (the prefix below dense_base is range A)."""
    regime = ("R2", "R1", "R4")[(T + Hq) % 3]
    tail = Hq == 28
    c, pre = build(regime, 2 if tail else 1, T, Hq=Hq, Hkv=Hkv, n=20011, p=20079, C=1 if tail else None, tail=tail,
                   seed=Hq * 1000 + T)
    run_case(c, f"Hq{Hq} Hkv{Hkv} T{T} {regime}", M=22000, pre_spill=pre)


# ---- (c) split edges ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_empty_trailing_split(cuda_lib):
    """Dense layer, default layout, Hq 8, Hkv 1, prefix 600, T = 1024: 64 m-blocks and 3 splits on a 132-SM H100; m-block 0's
    causal limit ends before its last split begins, so that CTA hands an empty state to the merge."""
    c, pre = build("R1", 1, 1024, Hq=8, Hkv=1, n=600, p=600, seed=7)
    sp = c.splits("dense")
    per = split_per(c.ntot(0, "dense"), sp)
    assert sp > 1 and (sp - 1) * per >= 600 + 16, f"no empty split ({sp} splits of {per})"
    run_case(c, "empty trailing split", M=4096, pre_spill=pre)


EDGES = [   # (label, Hq, Hkv, n, T): store lengths around a tile edge, one split, an empty store, a boundary in the chunk's rows
    ("n64k-1", 32, 8, 6399, 64), ("n64k", 32, 8, 6400, 64), ("n64k+1", 32, 8, 6401, 64),
    ("one-split-small-n", 32, 8, 300, 64), ("one-split-large-T", 32, 8, 5000, 1024), ("empty-store", 32, 8, 0, 128),
    ("boundary-in-chunk", 8, 8, 1000, 512),
]


@pytest.mark.gpu
@pytest.mark.parametrize("label,Hq,Hkv,n,T", EDGES, ids=[e[0] for e in EDGES])
def test_split_edges(cuda_lib, label, Hq, Hkv, n, T):
    c, pre = build("R1", 1, T, Hq=Hq, Hkv=Hkv, n=n, p=max(n, 64), seed=n + T)
    sp = c.splits("sparse")
    if label.startswith("one-split"):
        assert sp == 1
    if label == "boundary-in-chunk":
        per, base = split_per(c.ntot(0, "sparse"), sp), n + NS + NL
        assert any(base < s * per < base + T for s in range(1, sp)), f"{sp} splits of {per}: no boundary in the chunk"
    run_case(c, label, M=max(n, 64) + 2048, pre_spill=pre)


# ---- (d) captured plans --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3])
def test_captured_chunk_replays_read_the_replay_lengths(cuda_lib, B):
    """Capture plan_chunk(T) -> sparse -> dense once; replay; spill eagerly and replay; rewind part of the chunk and replay.
    Every replay against fp64 over the lengths of that replay.  The split count is the host's estimate at capture."""
    T, M, gen = 64, 20000, 300
    est = host_splits(T, 4, 8, B, sms(), M + NS + NL + gen)[1]
    kw = dict(C=1, spill=True, x=(40, 67, 101)) if B == 3 else {}
    c, pre = build("R1", B, T, n=2000, p=2000, seed=50 + B, splits=est, **kw)
    ctx = make_ctx(c, M, gen=gen, t_max=T)
    fill(ctx, c, pre)
    if c.spill:
        assert ctx.spill_window().tolist() == c.x
    # the eager split count, then the graph
    c.fixed_splits = None
    eager = run_chunk(ctx, c)
    assert eager["sparse"][2] == c.splits("sparse") and eager["dense"][2] == c.splits("dense")
    c.fixed_splits = est
    ctx.rewind(torch.full((B,), T, dtype=torch.int32, device=DEV))
    o1 = torch.empty((B, T, c.Hq * d), dtype=torch.bfloat16, device=DEV)
    o0 = torch.empty_like(o1)
    f1 = torch.empty((B * T * c.Hq, d), dtype=torch.float32, device=DEV)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        ctx.plan_chunk(T)
        ctx.chunk_attend(1, T, c.q, c.k, c.v, o1)
        f1.copy_(ctx.last_out_f32())
        ctx.chunk_attend(0, T, c.q, c.k, c.v, o0)
    captured = ctx.get_info("chunk_splits")
    assert captured == est and est != eager["sparse"][2] and est != eager["dense"][2], \
        f"captured {captured} splits, estimate {est}, eager {eager['sparse'][2]} / {eager['dense'][2]}"

    def replay(label, capture_check=False):
        for layer in ("sparse", "dense"):
            c.check_inputs(layer, capture=capture_check)
        graph.replay()
        torch.cuda.synchronize()
        check_out(c, o1, f1, c.restate("sparse", splits=captured), f"{label} sparse")
        check_out(c, o0, ctx.last_out_f32(), c.restate("dense", splits=captured), f"{label} dense")
        c.commit([T] * B)

    replay("replay")
    c.stale_n = [k.shape[1] for k in c.store_k]
    spilled = ctx.spill_window().tolist()
    assert spilled == c.do_spill()
    replay("replay after spill", capture_check=True)
    drop = [T // 2 + 7 * b for b in range(B)]
    ctx.rewind(torch.tensor(drop, dtype=torch.int32, device=DEV))
    for b in range(B):   # the rewind keeps T - drop[b] rows of the last replay
        c.win_k[b], c.win_v[b] = c.win_k[b][:, :c.win_k[b].shape[1] - drop[b]], c.win_v[b][:, :c.win_v[b].shape[1] - drop[b]]
        c.dk[b], c.dv[b] = c.dk[b][:c.dk[b].shape[0] - drop[b]], c.dv[b][:c.dv[b].shape[0] - drop[b]]
    replay("replay after rewind")
    assert ctx.error_flags() == 0


# ---- (e) ticket reuse ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_back_to_back_launches_reuse_the_tickets(cuda_lib):
    """Four chunk steps of 64, 256, 37, 128 tokens, each on the sparse then the dense layer: eight chunk_attend launches with no
    synchronisation between them over one partial scratch and one set of tickets, each launch at another split count than the
    one before (16, 3, 4, 3, 16, 3, 8, 3 on 132 SMs: the dense cache is short enough that 512 keys per split binds) and the
    steps at 2, 8, 2, 4 m-blocks.  Every launch's inputs are self-checked first; its bf16 output against fp64 (the fp32 bar plus
    the bf16 rounding of the element)."""
    Ts = (64, 256, 37, 128)
    c, _ = ticket_case(Ts, sms())
    pre = snapshot(c)
    refs = []
    chk = _copy(c)
    for T in Ts:
        _step_view(chk, c, T)
        for layer in ("sparse", "dense"):
            refs.append((chk.splits(layer), chk.check_inputs(layer)[0]))
        chk.commit([T])
    ctx = make_ctx(c, 32000, gen=1100, t_max=max(Ts))
    fill(ctx, c, pre)
    q, k, v = c.q, c.k, c.v
    outs, counts = [], []
    for T in Ts:
        ctx.plan_chunk(T)
        for layer in (1, 0):
            outs.append(ctx.chunk_attend(layer, T, q[:, :T].contiguous(), k[:, :T].contiguous(), v[:, :T].contiguous()))
            counts.append(ctx.get_info("chunk_splits"))
    torch.cuda.synchronize()
    assert counts == [sp for sp, _ in refs], f"chunk_splits {counts}, host formula {[sp for sp, _ in refs]}"
    assert all(a != b for a, b in zip(counts, counts[1:])), f"consecutive launches share a split count: {counts}"
    for i, (out, (sp, o)) in enumerate(zip(outs, refs)):
        got = out.reshape(o.shape).double()
        err = (got - o).abs() - 2.0 ** -8 * o.abs()
        worst = float((err.amax(-1) / o.abs().amax(-1)).max())
        assert worst <= BAR, f"launch {i} (T={Ts[i // 2]}, {('sparse', 'dense')[i % 2]}, {sp} splits): {worst:.3e}"
    assert ctx.error_flags() == 0


def _copy(c):
    """A view of case c whose lengths advance on their own (commit() replaces list entries, never the tensors in place)."""
    import copy
    v = copy.copy(c)
    v.win_k, v.win_v, v.dk, v.dv, v.tails = list(c.win_k), list(c.win_v), list(c.dk), list(c.dv), list(c.tails)
    return v


def _step_view(v, c, T):
    v.T, v.q, v.k, v.v = T, c.q[:, :T], c.k[:, :T], c.v[:, :T]


def ticket_case(Ts, n_sms, dev=DEV):
    """The ticket-reuse case: 30 000 store keys, a 1 500-row dense cache, one request; the tile at every launch's checked split
    boundary carries mass (planted before the fill, at the lengths each step will have)."""
    c = Case("R1", 1, max(Ts), n=30000, p=1500, seed=77, sms=n_sms, dev=dev)
    sim, tiles = _copy(c), []
    for T in Ts:
        _step_view(sim, c, T)
        tiles += [(layer, sim.boundary(0, layer), sim._lse(layer)) for layer in ("sparse", "dense")]
        sim.commit([T])
    for layer, k0, _ in tiles:   # every tile as strong as the last step needs, so that no later tile hides an earlier one
        lse = max(x for ly, _, x in tiles if ly == layer)
        if c._in_a_or_dense(0, layer, k0, CK_KT):
            c._set_key(0, layer, k0, c._along(lse + math.log(0.5 / CK_KT), 0.25, CK_KT))
    return c, sim
