"""Long generation against fp64 at the long-generation lines' shapes (`-m gpu`).

1. The shared line: Llama-3.1-8B heads (Hq 32, Hkv 8), K10 L150, B = 8 requests forked from one 98 000-token prompt in one slot,
   max_length 131 072, generation_buffer 256, shared spill, dense_tail_rows R = 4 400.  The module's fixture reaches the line's
   state through the library's own calls: request 0 filled, forked to the others, then about 4 100 tokens per request in 4-token
   chunk steps with ragged per-request rewinds, two 40-token chunk steps checked against fp64, and a spill (keep 48) whenever the next step does not fit
   the fullest window -- 16 spills.  The tails end on and next to 32-row tile edges (4 064, 4 095, 4 096, 4 097, 4 127, 4 128)
   and request 5 ends at R - 8, so that the 8-node tree takes it to exactly R.  The host mirrors every request's window, tail and
   private runs.  Checked:
     * the chunk steps against fp64 over the prompt rows below dense_base, the request's tail (thousands of rows) and the chunk;
     * the sparse store (prompt bitwise unchanged, every spilled run bitwise where the spill order puts it), the visibility map,
       and the tables against a fresh build over every stored key;
     * a sparse step (three-launch path) with queries near keys of each request's first and last spill, against fp64 over the
       prompt, the request's own private keys and its window;
     * dense steps over the long tails -- T = 1 (chunks of 8 members), a T = 4 chain (chunks of 2), the 8-node tree (chunks of 1)
       -- against fp64 over the prompt, the request's own tail and the visible step rows, the bf16 output the fp32 output rounded
       half-up; on a 132-SM H100 the T = 1 step's work items include one wholly inside a member's tail and one that starts inside
       a tail;
     * after a fork over request 2 from request 5, a sparse and a dense step: request 2 sees 5's tail and private runs only.
2. The single-request line: B = 1, 98 000-token prompt, max_length 102 208 (two key segments of 51 136), exclusive spill, 16
   spills of 256 keys into segment 1; the tables against a rebuild, then the fused kernel (fused_kreg 0 and 1) against fp64 with
   queries near first- and last-spill keys, nnz and lists exact.

Regimes: the sparse store is R1 (key mean); the dense check steps run R2 (the tails take >= 90 % of the mass) and R4 (queries x 16,
the dominant row deep in each tail).  Before any library call each check shows that its named perturbations move the fp64 output
by >= 10x the 1e-3 bar.  tests/test_long_gen_numerics_inputs_cpu.py runs the same schedule, generators and self-checks without a
GPU.
"""
import pytest
import torch

from tests.support.fp64 import BAR, SIMHASH_EPS, assert_rounded_half_up, key_codes, rel_rows, restate
from tests.support.library import (DEV, NL, NS, assert_tables_equal, d, lsh_tables, skip_unless_132_sms,
                                   two_layer_context)
from tests.support.long_gen import (DenseTails, PrivateRuns, check_dense_tails, restate_chunk, schedule, tail_items)
from tests.support.sparse_cases import (GEN, HKV, HQ, KK, LL, M_LONG, N_C2, TREE, check_codes_lists, check_outputs,
                                        make_batch, seed_of, step)

pytestmark = pytest.mark.gpu
B, P, R = 8, 98000, 4400
TAILS = (4096, 4095, 4097, 4128, 4127, 4392, 4064, 4100)   # tokens each request commits; request 5 ends at R - 8
T_GEN, KEEP, CHUNK_AT, T_CHUNK = 4, NL - 16, (2000, 3500), 40
DOM_AT = tuple(2000 + 41 * b for b in range(B))              # tail row of each request's dominant dense key
SPILLS = 16
bits = lambda x: x.contiguous().view(torch.int16)   # noqa: E731


def _cat_window(win, rows):
    """Window (Hkv, w, d) + rows (n, Hkv, d)."""
    return torch.cat([win, rows.transpose(0, 1)], dim=1)


def generate(ctx, c, runs, dt, events, priv, seed):
    """Drive ctx through the schedule's events, mirroring windows, tails and private runs; chunk steps are checked against
    fp64 as they run.  Returns one (worst error, ignores_tail margin) per chunk step."""
    st = c["slots"][0]
    g = torch.Generator(device=DEV).manual_seed(seed)
    rnd = lambda *s: torch.randn(s, generator=g, device=DEV, dtype=torch.float64)   # noqa: E731
    chunks = []
    for kind, x in events:
        if kind == "spill":
            assert ctx.spill_window(KEEP).tolist() == x
            runs.spill(x)
            for b in range(B):   # a slot's new keys go in request order; each request keeps its sinks and newest KEEP rows
                priv.append((c["win_k"][b][:, NS:NS + x[b]], c["win_v"][b][:, NS:NS + x[b]]))
                c["win_k"][b] = torch.cat([c["win_k"][b][:, :NS], c["win_k"][b][:, NS + x[b]:]], dim=1)
                c["win_v"][b] = torch.cat([c["win_v"][b][:, :NS], c["win_v"][b][:, NS + x[b]:]], dim=1)
            continue
        n = T_GEN if kind == "step" else T_CHUNK
        keep = [n - dr for dr in x]
        # sparse rows: token t of a step is one row plus a little noise per request, so that a query near one request's copy is
        # near the other requests' copies too (a request that saw another's private keys would attend to them)
        ks = (rnd(1, n, HKV, d) + st["mu"].reshape(1, 1, HKV, d) + 0.3 * rnd(B, n, HKV, d)).bfloat16()
        vs = torch.randn((B, n, HKV, d), generator=g, device=DEV).bfloat16()
        qs = torch.randn((B, n, HQ, d), generator=g, device=DEV).bfloat16()
        dk, dv = dt.step_rows(n, keep)
        if kind == "step":   # (the sparse T-token decode does not run B = 8 over two key segments: chunk steps append the rows)
            ctx.plan_chunk(n)
            ctx.chunk_attend(1, n, qs, ks, vs)
            ctx.chunk_attend(0, n, qs, dk, dv)
        else:
            qd = dt.check_step("R2", n, HQ)[0]
            o = restate_chunk(dt, qd, dk, dv)
            moved = rel_rows(restate_chunk(dt, qd, dk, dv, "ignores_tail"), o)
            assert moved >= 10 * BAR, f"chunk: ignoring the tail moves the output by {moved:.2e} only"
            ctx.plan_chunk(n)
            ctx.chunk_attend(1, n, qs, ks, vs)
            out = ctx.chunk_attend(0, n, qd, dk, dv)
            o32 = ctx.last_out_f32()
            worst = rel_rows(o32.reshape(B, n, HQ, d), o)
            assert_rounded_half_up(out, o32, "dense chunk")
            chunks.append((min(dt.tl), worst, moved))
        ctx.rewind(torch.tensor(x, dtype=torch.int32, device=DEV))
        dt.commit(dk, dv, keep)
        for b in range(B):
            c["win_k"][b] = _cat_window(c["win_k"][b], ks[b, :keep[b]] - st["avg"])
            c["win_v"][b] = _cat_window(c["win_v"][b], vs[b, :keep[b]])
    return chunks


@pytest.fixture(scope="module")
def state(cuda_lib):
    c = make_batch("R1", 1, n=N_C2, lens=(NS + 1,), seed=seed_of("long gen"))   # the prompt's store; a window of NS sinks
    c.update(B=B, slot_of=[0] * B, win_k=[c["win_k"][0].clone() for _ in range(B)],
             win_v=[c["win_v"][0].clone() for _ in range(B)])
    st = c["slots"][0]
    ctx = two_layer_context(KK, LL, HQ, HKV, B, M_LONG, GEN, c["hf"], dict(decode_impl=1, save_mask=1, out_f32=1),
                            max_query_tokens=8, num_contexts=1, shared_spill=True, dense_tail_rows=R, alloc_dense_kv=True)
    ctx.reserve_chunk_tokens(T_CHUNK)
    dt = DenseTails(B, P, R, HKV, DOM_AT, seed_of("long gen dense"), DEV)
    ctx.attn_fill(1, 0, st["key"], st["value"], st["kn"])
    ctx.lsh_build(1, 0, st["kcodes"])
    ctx.window_fill(1, 0, st["avg"].contiguous(), c["win_k"][0].contiguous(), c["win_v"][0].contiguous())
    ctx.dense_fill(0, 0, dt.dk, dt.dv, P)
    for b in range(1, B):
        ctx.fork(0, b)
    events, _ = schedule(TAILS, T_GEN, NS, NS + NL + GEN, KEEP, CHUNK_AT, T_CHUNK)
    assert sum(e[0] == "spill" for e in events) == SPILLS
    runs, priv = PrivateRuns(B, N_C2), []
    chunks = generate(ctx, c, runs, dt, events, priv, seed=seed_of("long gen steps"))
    assert ctx.error_flags() == 0
    assert dt.tl == list(TAILS)
    for tl, worst, moved in chunks:
        print(f"chunk over tails >= {tl} rows: ignores_tail moves the output by {moved:.2e}; "
              f"largest relative head error {worst:.2e} ({worst / BAR:.1%} of the bar)")
    prompt = dict(st)
    k_st, v_st, kn_st = ctx.read_cache(1)
    total = runs.total
    theirs = ctx.hash_keys(k_st[0, :, N_C2:total].contiguous())   # the codes the spills merged into the tables
    # the restatements of the steps read the whole store
    st.update(key=k_st[0, :, :total], value=v_st[0, :, :total], kn=kn_st[0, :, :total], kcodes=torch.cat([st["kcodes"], theirs], -1))
    yield dict(ctx=ctx, c=c, dt=dt, runs=runs, priv=priv, chunks=chunks, prompt=prompt, theirs=theirs)
    del ctx


def test_chunks_over_long_tails(state):
    """The two chunk steps, run over tails of about 2 000 and 3 500 rows, within the bar (checked as they ran)."""
    assert len(state["chunks"]) == 2 and min(tl for tl, _, _ in state["chunks"]) >= 1900
    for tl, worst, _ in state["chunks"]:
        assert worst <= BAR, f"chunk over tails of >= {tl} rows: fp32 output differs from fp64 by {worst:.3e}"


def test_store_visibility_and_tables(state):
    """After 16 spills: the prompt's records and norms unchanged, each run bitwise where the spill order puts it, the visibility
    map the expected interleaving, the tables equal to a fresh build over every stored key (as sets per bucket)."""
    ctx, c, runs, pr = state["ctx"], state["c"], state["runs"], state["prompt"]
    n, total = N_C2, runs.total
    assert total == n + sum(k.shape[1] for k, _ in state["priv"]) and total <= M_LONG
    k_st, v_st, kn_st = (x[0, :, :total] for x in ctx.read_cache(1))
    assert torch.equal(bits(k_st[:, :n]), bits(pr["key"])) and torch.equal(bits(v_st[:, :n]), bits(pr["value"])), \
        "the spills changed the prompt's records"
    assert torch.equal(kn_st[:, :n], pr["kn"]), "the spills changed the prompt's key norms"
    off = n
    for i, (mk, mv) in enumerate(state["priv"]):
        w = mk.shape[1]
        assert torch.equal(bits(k_st[:, off:off + w]), bits(mk)), f"run {i}: spilled keys"
        assert torch.equal(bits(v_st[:, off:off + w]), bits(mv)), f"run {i}: spilled values"
        kn, norm = kn_st[:, off:off + w], mk.double().norm(dim=-1)
        assert torch.equal(kn.bfloat16().float(), kn) and bool(((kn.double() - norm).abs() <= 2.0 ** -8 * norm).all()), \
            f"run {i}: spilled key norms"
        off += w
    assert all(len(r) == 16 for r in runs.runs), "every request spilled at every spill"
    vis = ctx.visibility()[0, :total - n]
    assert torch.equal(vis, runs.visibility(M_LONG, DEV)[:total - n]), "visibility map"
    rows = k_st[:, n:total].contiguous()
    ours, theirs = key_codes(rows, c["hf"], KK, LL), state["theirs"]
    bad = torch.nonzero(ours != theirs)
    if bad.shape[0]:   # the context's key hash may differ from fp64 only within rounding of a zero projection
        kk = rows[bad[:, 0], bad[:, 2]].double()
        cols = bad[:, 1, None] * KK + torch.arange(KK, device=DEV)[None]
        margin = (c["hf"].double().t()[cols] * kk[:, None]).sum(-1).abs().min(dim=-1).values
        assert float(margin.max()) < SIMHASH_EPS * float(rows.float().norm(dim=-1).mean()), float(margin.max())
    ref = two_layer_context(KK, LL, HQ, HKV, B, M_LONG, GEN, c["hf"], num_contexts=1, shared_spill=True)
    ref.lsh_build(1, 0, torch.cat([pr["kcodes"], theirs], -1).contiguous())
    assert_tables_equal(lsh_tables(ctx, 1), lsh_tables(ref, 1))


def sparse_step(state, label, seed):
    """One sparse step (three-launch path) with queries near keys of each request's first spill (even kv-groups) and last
    spill (odd kv-groups), against fp64; the private-key filter and the key mean must move every request by >= 10x the bar.
    The step is rewound afterwards."""
    ctx, c, runs = state["ctx"], state["c"], state["runs"]
    st = c["slots"][0]
    g = torch.Generator(device=DEV).manual_seed(seed)
    near = torch.stack([torch.stack([st["key"][h, runs.runs[b][0 if h % 2 == 0 else -1][0] + 3] for h in range(HKV)])
                        for b in range(B)]).double()                                              # (B, Hkv, d)
    c["q"] = (near.repeat_interleave(c["G"], 1)[:, None]
              + 0.25 * torch.randn((B, 1, HQ, d), generator=g, device=DEV, dtype=torch.float64)).bfloat16()
    c["k_new"] = (torch.randn((B, 1, HKV, d), generator=g, device=DEV, dtype=torch.float64)
                  + st["mu"].reshape(1, 1, HKV, d)).bfloat16()
    c["v_new"] = torch.randn((B, 1, HKV, d), generator=g, device=DEV).bfloat16()
    c["vis"] = runs.masks(runs.runs, DEV)
    rr = step(ctx, c)
    assert rr["fused"] == 0, f"{label}: last_decode_fused = {rr['fused']}"
    sets = check_codes_lists(c, rr)
    o = restate(c, rr["codes"], sets=sets)[0]
    moved = {"uncentred": rel_rows(restate(c, rr["codes"], "uncentred", sets=sets)[0], o)}
    own = c["vis"]
    everyone = [r for rs in runs.runs for r in rs]
    for name, other in (("sees_all_private", [everyone] * B), ("sees_no_private", [[]] * B)):
        c["vis"] = runs.masks(other, DEV)
        alt = restate(c, rr["codes"])[0]
        moved[name] = min(rel_rows(alt[b], o[b]) for b in range(B))
    c["vis"] = own
    print(f"{label}: perturbations move every request by " + ", ".join(f"{k} {v:.2e}" for k, v in moved.items()))
    for name, m in moved.items():
        assert m >= 10 * BAR, f"{label}: '{name}' moves a request by {m:.2e} only"
    check_outputs(c, rr, sets, label)
    for b in range(B):
        listed = rr["res"][b, 0][torch.arange(rr["res"].shape[-1], device=DEV)[None] < rr["nnz"][b, 0][:, None]]
        assert bool((listed >= N_C2).any()), f"{label}: request {b} sampled none of its spilled keys"
    ctx.rewind(torch.ones(B, dtype=torch.int32, device=DEV))


def test_sparse_step(state):
    sparse_step(state, "long gen sparse B8", 11)


def dense_step(state, label, regime, T, tree=False):
    """One dense step over the long tails against fp64, after the regime's self-checks; undone afterwards."""
    ctx, dt = state["ctx"], state["dt"]
    q, k, v = dt.check_step(regime, T, HQ)
    parents = [TREE] * B if tree else None
    o, moved = check_dense_tails(dt, regime, q, k, v, parents)
    if T == 1:
        ctx.plan()
        out = ctx.dense_decode(0, q[:, 0].contiguous(), k[:, 0].contiguous(), v[:, 0].contiguous())
    else:
        ctx.plan(T, parents=torch.tensor(parents, dtype=torch.int32, device=DEV) if tree else None)
        out = ctx.dense_decode_tokens(0, T, q, k, v)
    o32 = ctx.last_out_f32()
    assert ctx.error_flags() == 0
    worst = rel_rows(o32.reshape(B, T, HQ, d), o)
    print(f"{label}: perturbations " + ", ".join(f"{a} {b:.2e}" for a, b in moved.items())
          + f"; largest relative head error {worst:.2e} ({worst / BAR:.1%} of the bar)")
    assert worst <= BAR, f"{label}: fp32 output differs from fp64 by {worst:.3e} relative"
    assert_rounded_half_up(out, o32, label)
    if tree:
        ctx.accept(torch.zeros((B, T), dtype=torch.int32, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV))
    else:
        ctx.rewind(torch.full((B,), T, dtype=torch.int32, device=DEV))


@pytest.mark.parametrize("regime", ["R2", "R4"])
@pytest.mark.parametrize("shape", ["T1", "T4", "tree8"])
def test_dense_steps(state, shape, regime):
    """T = 1 (one chunk of 8 members), a T = 4 chain (chunks of 2), the 8-node tree (chunks of 1; request 5's tail reaches
    exactly R)."""
    T = {"T1": 1, "T4": 4, "tree8": 8}[shape]
    dense_step(state, f"long gen dense {shape} {regime}", regime, T, tree=shape == "tree8")


def test_dense_partition_reaches_tails(state):
    """dense_partition_of's items of the T = 1 step on a 132-SM H100 (8 warps per CTA): at least one lies wholly inside one
    member's tail and at least one starts inside a tail."""
    skip_unless_132_sms()
    inside, boundary = tail_items(P, [t + 1 for t in state["dt"].tl], 1, HQ // HKV, HKV, 132 * 8)
    print(f"T = 1 step: {inside} items inside a tail, {boundary} items starting inside a tail")
    assert inside >= 1 and boundary >= 1


def test_after_fork(state):
    """fork(5, 2) after the 16 spills: request 2 continues request 5 -- its tail, its window and the private runs it sees --
    and sees none of its own old runs.  A sparse and a dense step against fp64."""
    ctx, c, dt, runs = state["ctx"], state["c"], state["dt"], state["runs"]
    ctx.fork(5, 2)
    runs.fork(5, 2)
    dt.fork(5, 2)
    c["win_k"][2], c["win_v"][2] = c["win_k"][5].clone(), c["win_v"][5].clone()
    assert torch.equal(ctx.visibility()[0, :runs.total - N_C2], runs.visibility(M_LONG, DEV)[:runs.total - N_C2])
    sparse_step(state, "after fork sparse B8", 12)
    dense_step(state, "after fork dense T1 R2", "R2", 1)


# ---- 2. the single-request line -----------------------------------------------------------------------------------------
M_ONE = 102208


@pytest.mark.parametrize("kreg", [0, 1])
def test_single_request_line(cuda_lib, kreg):
    """B = 1, exclusive spill, 16 spills of 256 keys into key segment 1, then the fused kernel against fp64 with queries near
    keys of the first and the last spill."""
    c = make_batch("R1", 1, n=N_C2, lens=(NS + NL + 1,), seed=seed_of("long gen one"))
    st = c["slots"][0]
    ctx = two_layer_context(KK, LL, HQ, HKV, 1, M_ONE, GEN, c["hf"], dict(decode_impl=1, fused_kreg=kreg, save_mask=1, out_f32=1),
                            max_query_tokens=8)
    S = ctx.get_info("table_segments")
    seg = (((M_ONE + S - 1) // S) + 63) & ~63
    if torch.cuda.get_device_properties(0).multi_processor_count == 132:
        assert (S, seg) == (2, 51136), (S, seg)
    ctx.attn_fill(1, 0, st["key"], st["value"], st["kn"])
    ctx.lsh_build(1, 0, st["kcodes"])
    ctx.window_fill(1, 0, st["avg"].contiguous(), c["win_k"][0].contiguous(), c["win_v"][0].contiguous())
    g = torch.Generator(device=DEV).manual_seed(5)
    keys, vals = [st["key"]], [st["value"]]
    for _ in range(16):
        for _ in range(GEN // 8):
            k = (torch.randn((1, 8, HKV, d), generator=g, device=DEV, dtype=torch.float64) + st["mu"].reshape(1, 1, HKV, d)).bfloat16()
            v = torch.randn((1, 8, HKV, d), generator=g, device=DEV).bfloat16()
            ctx.plan(8)
            ctx.decode_tokens(1, 8, torch.randn((1, 8, HQ, d), generator=g, device=DEV).bfloat16(), k, v)
            c["win_k"][0] = _cat_window(c["win_k"][0], k[0] - st["avg"])
            c["win_v"][0] = _cat_window(c["win_v"][0], v[0])
        assert ctx.spill_window().tolist() == [GEN]
        keys.append(c["win_k"][0][:, NS:NS + GEN])
        vals.append(c["win_v"][0][:, NS:NS + GEN])
        c["win_k"][0] = torch.cat([c["win_k"][0][:, :NS], c["win_k"][0][:, NS + GEN:]], dim=1)
        c["win_v"][0] = torch.cat([c["win_v"][0][:, :NS], c["win_v"][0][:, NS + GEN:]], dim=1)
    assert ctx.error_flags() == 0
    total = N_C2 + 16 * GEN
    assert N_C2 >= seg, "the spilled keys are not all in key segment 1"
    k_st, v_st, kn_st = ctx.read_cache(1)
    assert torch.equal(bits(k_st[0, :, :total]), bits(torch.cat(keys, 1))), "stored keys"
    assert torch.equal(bits(v_st[0, :, :total]), bits(torch.cat(vals, 1))), "stored values"
    theirs = ctx.hash_keys(k_st[0, :, N_C2:total].contiguous())
    ref = two_layer_context(KK, LL, HQ, HKV, 1, M_ONE, GEN, c["hf"])
    ref.lsh_build(1, 0, torch.cat([st["kcodes"], theirs], -1).contiguous())
    assert_tables_equal(lsh_tables(ctx, 1), lsh_tables(ref, 1))
    del ref
    st.update(key=k_st[0, :, :total], value=v_st[0, :, :total], kn=kn_st[0, :, :total], kcodes=torch.cat([st["kcodes"], theirs], -1))
    c["n"] = total
    near = torch.stack([st["key"][h, N_C2 + 3 if h % 2 == 0 else total - GEN + 3] for h in range(HKV)]).double()
    c["q"] = (near.repeat_interleave(c["G"], 0)[None, None]
              + 0.25 * torch.randn((1, 1, HQ, d), generator=g, device=DEV, dtype=torch.float64)).bfloat16()
    c["k_new"] = (torch.randn((1, 1, HKV, d), generator=g, device=DEV, dtype=torch.float64) + st["mu"].reshape(1, 1, HKV, d)).bfloat16()
    c["v_new"] = torch.randn((1, 1, HKV, d), generator=g, device=DEV).bfloat16()
    r = step(ctx, c)
    assert r["fused"] == 1, f"last_decode_fused = {r['fused']}"
    sets = check_codes_lists(c, r)
    o = restate(c, r["codes"], sets=sets)[0]
    for name in ("uncentred", "drop_sampled"):
        moved = rel_rows(restate(c, r["codes"], name, sets=sets)[0], o)
        print(f"single request kreg{kreg}: {name} moves the output by {moved:.2e}")
        assert moved >= 10 * BAR, f"'{name}' moves the output by {moved:.2e} only"
    check_outputs(c, r, sets, f"single request kreg{kreg}")
    listed = r["res"][0, 0][torch.arange(r["res"].shape[-1], device=DEV)[None] < r["nnz"][0, 0][:, None]]
    assert bool((listed >= N_C2 + (16 - 1) * GEN).any()) and bool(((listed >= N_C2) & (listed < N_C2 + GEN)).any()), \
        "the step sampled no key of the first or of the last spill"
