"""Batched decode over one long context against fp64, at the shapes the shared-context, beam and long-generation lines measure
(`-m gpu`).

Those lines run Llama-3.1-8B heads (Hq 32, Hkv 8, K10 L150) over one 98 K-token context at B = 1 ... 32.  The other fp64 file
(test_gpu_numerics.py) stops at B <= 4 and n <= 70 000 with one slot per request and equal window lengths, and the B = 8 test at
this size (test_gpu_shared.py::test_c2_size_b8_one_context) compares two contexts that run the same kernels.  Here every request
of a step is checked against an fp64 restatement of ITS slot's store and ITS own window:

  * the path each measured shape runs is pinned (test_measured_shapes_path): fused at B <= 4, the three-launch path
    (simhash -> probe -> stream-K attend) at B >= 8, the fused T-token kernel in several waves for T = 4;
  * one C2-size context (n = 97 932, M = 98 304, or 131 072 with shared spill) per slot, on the device; the key codes are an
    fp64 GEMM (`key_codes`) handed to lsh_build, so the tables do not depend on the key-hash kernel;
  * ragged windows (69, 150, 324, 200 rows cycled over the requests, 324 = the full window of generation_buffer 256), windows
    of 4 000 ... 4 172 rows, two documents on two slots, 1 024 heads in one step, T = 4 chains and an 8-node tree, a step after a
    shared spill and after a fork of a request that spilled, and the dense layers in shared-prefix mode at B = 8 and 32.

Regimes (the knobs of test_gpu_numerics.py): R1 key mean, R2 sinks (the window holds >= 90 % of the mass), R4 large logits with
one dominant row, either the LAST stored key (last key segment, last sampled tile) or the last window row of every request.
Before any library call each case checks that its named perturbations of the restatement move the output by >= 10x the 1e-3
bar: the regime's own (SELF_CHECK) and, for batches, `window_of_request_0` (every request attends over request 0's window) and,
with two slots whose stores carry the mass (R1, R4 with a dominant key), `wrong_document` (request b attends over the other
slot's store); in R1, where the sampled half carries nearly all the mass, `drop_sampled` must move EVERY checked head.  Fused
steps run with save_mask = 0, as the measured lines do, and take their codes and lists from a save_mask = 1 twin.
tests/test_batch_numerics_inputs_cpu.py runs the same generator and restatement at a reduced size without a GPU.

The fp64 work runs with torch on whichever device holds the case (IEEE fp64 tensor arithmetic, none of the library's kernels).
"""
import pytest
import torch

from magicpig_b200 import synth
from tests.support.fp64 import BAR, SIMHASH_EPS, assert_rounded_half_up, avg_of, key_codes, rel_rows, restate
from tests.support.library import DEV, NL, NS, d, skip_unless_132_sms, two_layer_context
from tests.support.sparse_cases import (GEN, HKV, HQ, KK, LENS, LL, M_C2, M_LONG, N_C2, TREE, batch_ctx, check_codes_lists,
                                        check_dense_inputs, check_inputs, check_outputs, make_batch, make_dense_slots, seed_of,
                                        step, twin_step)

LONG_GEN = 4104                       # generation_buffer of the long-generation line's "no spill" arm: windows of up to 4 172 rows
LONG_LENS = (4000, 4172, 4100, 4050)


# ---- 1. the path each measured shape runs --------------------------------------------------------------------------------
# (B, T, max_length, shared_spill): fused_applicable, fused_cluster_waves, last_decode_fused, tokens_cluster_waves (T > 1)
PATHS = [
    ((1, 1, M_C2, False), (1, 1, 1, None)),     # bench.py: 32 clusters of two 1024-thread CTAs
    ((2, 1, M_C2, False), (1, 1, 1, None)),
    ((4, 1, M_C2, False), (1, 1, 1, None)),     # 512-thread CTAs, two per SM
    ((8, 1, M_C2, False), (0, 0, 0, None)),     # three-launch: simhash -> probe -> attend_mma (stream-K)
    ((16, 1, M_C2, False), (0, 0, 0, None)),
    ((32, 1, M_C2, False), (0, 0, 0, None)),
    ((8, 1, M_LONG, True), (0, 0, 0, None)),    # beam and shared long-generation lines
    ((4, 4, M_C2, False), (1, 1, 1, 4)),        # verification: the fused T-token kernel, 128 resident clusters per wave
    ((8, 4, M_C2, False), (0, 0, 1, 8)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("shape,want", PATHS, ids=[f"B{s[0]}-T{s[1]}{'-spill' if s[3] else ''}" for s, _ in PATHS])
def test_measured_shapes_path(cuda_lib, shape, want):
    """Which sparse-layer path a step of each measured shape runs (Llama-3.1-8B heads, K10 L150, one slot)."""
    skip_unless_132_sms()
    B, T, M, spill = shape
    ctx = two_layer_context(KK, LL, HQ, HKV, B, M, GEN, max_query_tokens=T, num_contexts=1, shared_spill=spill)
    got = [ctx.get_info("fused_applicable"), ctx.get_info("fused_cluster_waves")]
    g = torch.Generator(device=DEV).manual_seed(B)
    ctx.set_hash_func(synth.make_hash_func(d, KK, LL, seed=1).to(DEV))
    key = torch.randn((HKV, 300, d), generator=g, device=DEV).bfloat16()
    ctx.attn_fill(1, 0, key, key, key.float().norm(dim=-1))
    ctx.lsh_build(1, 0, ctx.hash_keys(key))
    for b in range(1, B):
        ctx.fork(0, b)
    for b in range(B):
        ctx.window_fill(1, b, torch.zeros((HKV, d), dtype=torch.bfloat16, device=DEV), key[:, :NS + NL].contiguous(),
                        key[:, :NS + NL].contiguous())
    q = torch.randn((B, T, HQ, d), generator=g, device=DEV).bfloat16()
    kv = torch.randn((B, T, HKV, d), generator=g, device=DEV).bfloat16()
    if T == 1:
        ctx.plan()
        ctx.decode(1, q[:, 0].contiguous(), kv[:, 0].contiguous(), kv[:, 0].contiguous())
    else:
        ctx.plan(T)
        ctx.decode_tokens(1, T, q, kv, kv)
    got.append(ctx.get_info("last_decode_fused"))
    got.append(ctx.get_info("tokens_cluster_waves") if T > 1 else None)
    assert tuple(got) == want, f"B={B} T={T}: (applicable, waves, fused, token waves) = {tuple(got)}"


# ---- 2./3. sparse cases ----------------------------------------------------------------------------------------------------
def sparse_case(label, regime, B, C=1, lens=LENS, place="key", T=1, parents=None, heads=None, fused=True, M=M_C2, gen=GEN,
                kreg=0, n=N_C2):
    """Generate, self-check, run one step and check it.  Fused steps run as the measured lines run them, with save_mask = 0
    (the CTAs list their selection in the carved extra row buffers); their codes and lists come from a save_mask = 1 twin
    filled identically, which must sample the same counts.  The three-launch path always writes its lists."""
    c = make_batch(regime, B, C=C, n=n, T=T, lens=lens, place=place, seed=seed_of(label, regime, place, kreg), parents=parents)
    moved = check_inputs(c, parents, heads)
    print(f"{label}: perturbations move the output by " + ", ".join(f"{k} {v:.2e}" for k, v in moved.items()))
    r = twin_step(lambda save_mask: batch_ctx(c, C=0 if B == 1 else C, M=M, gen=gen, kreg=kreg, save_mask=save_mask, t_max=T),
                  c, label, parents, fused)
    sets = check_codes_lists(c, r)
    return check_outputs(c, r, sets, label, parents, heads)


@pytest.mark.gpu
@pytest.mark.parametrize("kreg", [0, 1])
@pytest.mark.parametrize("regime", ["R1", "R2", "R4"])
def test_bench_config(cuda_lib, regime, kreg):
    """bench.py's configuration: B = 1 at C2 with save_mask = 0 (the CTAs list their selection in the carved extra row
    buffers), a full 324-row window."""
    sparse_case(f"bench {regime} kreg{kreg}", regime, 1, lens=(324,), kreg=kreg)


@pytest.mark.gpu
def test_shared_two(cuda_lib):
    sparse_case("shared B2", "R1", 2, lens=(69, 324))


@pytest.mark.gpu
@pytest.mark.parametrize("kreg", [0, 1])
@pytest.mark.parametrize("regime", ["R2", "R4"])
def test_shared_four(cuda_lib, regime, kreg):
    """Four requests on one slot: the fused kernel in 512-thread CTAs, ragged windows."""
    sparse_case(f"shared B4 {regime} kreg{kreg}", regime, 4, kreg=kreg)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["R1", "R2", "R4"])
def test_shared_eight(cuda_lib, regime):
    """Eight requests on one slot: the three-launch path, ragged windows."""
    sparse_case(f"shared B8 {regime}", regime, 8, fused=False)


@pytest.mark.gpu
def test_two_documents(cuda_lib):
    """Two slots holding different documents, requests bound 0, 1, 0, 1, ...: each attends over its own slot's store."""
    sparse_case("two documents B8", "R1", 8, C=2, fused=False)


@pytest.mark.gpu
def test_wide_batch(cuda_lib):
    """B = 32 on one slot: 1 024 heads in one step, the stream-K attend kernel at its widest.  Every head's codes and lists;
    fp64 outputs on four heads per request (rotating over the kv-groups), 128 heads.  R1: the sampled half carries nearly all of
    every head's mass, and dropping it must move every checked head by 10x the bar, so a lost or misweighted part shows."""
    heads = torch.zeros((32, HQ), dtype=torch.bool)
    for b in range(32):
        heads[b, [(b + 9 * j) % HQ for j in range(4)]] = True
    sparse_case("wide B32", "R1", 32, heads=heads, fused=False)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("regime,place", [("R2", "key"), ("R4", "win")], ids=["R2", "R4win"])
def test_long_windows(cuda_lib, regime, place, B):
    """generation_buffer 4 104: windows of 4 000 ... 4 172 rows (R2: the sinks thousands of rows before the query; R4: the
    dominant row in each window's last tile)."""
    lens = (4172,) if B == 1 else LONG_LENS
    sparse_case(f"long windows B{B} {regime}", regime, B, lens=lens, place=place, gen=LONG_GEN, fused=(B == 1))


@pytest.mark.gpu
@pytest.mark.parametrize("tree", [False, True], ids=["chain4", "tree8"])
def test_verification(cuda_lib, tree):
    """B = 8, a T = 4 chain or an 8-node tree after plan(T): every token against fp64 under the causal / ancestor mask, ragged
    windows; the fused T-token kernel in several waves."""
    T, parents = (8, [TREE] * 8) if tree else (4, None)
    sparse_case(f"verification B8 {'tree8' if tree else 'T4'}", "R2" if tree else "R4", 8, T=T, parents=parents)


# ---- after a shared spill ---------------------------------------------------------------------------------------------------
SPILLED = (40, 67, 101, 133, 170, 199, 230, 255)   # rows each request moves into the slot (window = NS + NL + these)


@pytest.mark.gpu
def test_after_shared_spill(cuda_lib):
    """B = 8 on one slot with shared_spill at the long-generation geometry (M = 131 072, generation_buffer 256).  Every request
    has grown its window by a different number of tokens (40 ... 255), decodes a step, spills; then a step with queries near
    its own spilled keys, a fork of a request that spilled, and one more step.  Each request against fp64 over the prompt, the
    private keys IT spilled and its remaining window.  The spilled rows are read back; their fp64 codes may differ from the
    codes the spill merged into the tables only where a projection is within rounding of zero, and the lists are restated
    over the merged codes."""
    B = 8
    c = make_batch("R1", B, lens=tuple(NS + NL + x for x in SPILLED), seed=seed_of("spill"))
    # window row NS + 3 (spilled by every request) is one row plus a little noise per request: a query near a request's own
    # copy is near every other request's copy too, so a request that saw another's private keys would attend to them
    gr = torch.Generator(device=DEV).manual_seed(4)
    for b in range(B):
        c["win_k"][b][:, NS + 3] = (c["win_k"][0][:, NS + 3].double()
                                    + 0.3 * torch.randn((HKV, d), generator=gr, device=DEV, dtype=torch.float64)).bfloat16()
    check_inputs(c)
    ctx = batch_ctx(c, M=M_LONG, shared_spill=True)
    r = step(ctx, c)
    assert r["fused"] == 0
    check_outputs(c, r, check_codes_lists(c, r), "before spill B8")
    for b in range(B):   # the step's token joins the window
        c["win_k"][b] = torch.cat([c["win_k"][b], (c["k_new"][b, 0] - avg_of(c, b))[:, None]], dim=1)
        c["win_v"][b] = torch.cat([c["win_v"][b], c["v_new"][b, 0][:, None]], dim=1)
    got = ctx.spill_window()
    assert got.tolist() == list(SPILLED)
    n, st = c["n"], c["slots"][0]
    total = n + sum(SPILLED)
    k_st, v_st, kn_st = ctx.read_cache(1)
    bits = lambda x: x.contiguous().view(torch.int16)   # noqa: E731
    assert torch.equal(bits(k_st[0, :, :n]), bits(st["key"])) and torch.equal(bits(v_st[0, :, :n]), bits(st["value"])), \
        "the spill changed the prompt's records"
    assert torch.equal(kn_st[0, :, :n], st["kn"]), "the spill changed the prompt's key norms"
    off = n
    for b in range(B):   # a slot's new keys go in request order; each request keeps its sinks and newest NL rows
        mk, mv = c["win_k"][b][:, NS:NS + SPILLED[b]], c["win_v"][b][:, NS:NS + SPILLED[b]]
        assert torch.equal(bits(k_st[0, :, off:off + SPILLED[b]]), bits(mk)), f"request {b}: spilled keys"
        assert torch.equal(bits(v_st[0, :, off:off + SPILLED[b]]), bits(mv)), f"request {b}: spilled values"
        kn = kn_st[0, :, off:off + SPILLED[b]]   # bf16(||k||) widened to fp32, as fill() stores
        norm = mk.double().norm(dim=-1)
        assert torch.equal(kn.bfloat16().float(), kn) and bool(((kn.double() - norm).abs() <= 2.0 ** -8 * norm).all()), \
            f"request {b}: spilled key norms"
        off += SPILLED[b]
        c["win_k"][b] = torch.cat([c["win_k"][b][:, :NS], c["win_k"][b][:, NS + SPILLED[b]:]], dim=1)
        c["win_v"][b] = torch.cat([c["win_v"][b][:, :NS], c["win_v"][b][:, NS + SPILLED[b]:]], dim=1)
    # the spilled keys' codes: fp64 from the rows read back; the tables hold the context's own hash of them, which may differ
    # only within rounding of a zero projection
    rows = k_st[0, :, n:total].contiguous()
    ours, theirs = key_codes(rows, c["hf"], KK, LL), ctx.hash_keys(rows)
    bad = torch.nonzero(ours != theirs)
    if bad.shape[0]:
        kk = rows[bad[:, 0], bad[:, 2]].double()
        cols = bad[:, 1, None] * KK + torch.arange(KK, device=DEV)[None]
        margin = (c["hf"].double().t()[cols] * kk[:, None]).sum(-1).abs().min(dim=-1).values
        assert float(margin.max()) < SIMHASH_EPS * float(rows.float().norm(dim=-1).mean()), float(margin.max())
    st.update(key=k_st[0, :, :total], value=v_st[0, :, :total], kn=kn_st[0, :, :total], kcodes=torch.cat([st["kcodes"], theirs], -1))
    spans, off = [], n
    for b in range(B):
        spans.append((off, off + SPILLED[b]))
        off += SPILLED[b]
    vis = [[s] for s in spans]
    g = torch.Generator(device=DEV).manual_seed(3)

    def masks(spans_of):
        out = []
        for b in range(B):
            m = torch.zeros(total, dtype=torch.bool, device=DEV)
            m[:n] = True
            for lo, hi in spans_of[b]:
                m[lo:hi] = True
            out.append(m)
        return out

    def private_step(label):
        c["vis"] = masks(vis)
        # queries near one of the request's own spilled keys, so that private keys are sampled
        near = torch.stack([st["key"][:, vis[b][0][0] + 3] for b in range(B)]).double()          # (B, Hkv, d)
        c["q"] = (near.repeat_interleave(c["G"], 1)[:, None] + 0.25 * torch.randn((B, 1, HQ, d), generator=g, device=DEV,
                                                                                   dtype=torch.float64)).bfloat16()
        c["k_new"] = (torch.randn((B, 1, HKV, d), generator=g, device=DEV, dtype=torch.float64)
                      + torch.stack([st["mu"]] * B).reshape(B, 1, HKV, d)).bfloat16()
        c["v_new"] = torch.randn((B, 1, HKV, d), generator=g, device=DEV).bfloat16()
        rr = step(ctx, c)
        assert rr["fused"] == 0, f"{label}: last_decode_fused = {rr['fused']}"
        sets = check_codes_lists(c, rr)
        # the private-key filter is visible: seeing every request's spilled keys, or none of its own, moves each request
        o = restate(c, rr["codes"], sets=sets)[0]
        own = c["vis"]
        for name, other in (("sees_all_private", masks([spans] * B)), ("sees_no_private", masks([[]] * B))):
            c["vis"] = other
            alt = restate(c, rr["codes"])[0]
            per_req = [rel_rows(alt[b], o[b]) for b in range(B)]
            assert min(per_req) >= 10 * BAR, f"{label}: '{name}' moves a request by {min(per_req):.2e} only"
            print(f"{label}: {name} moves every request by >= {min(per_req):.2e}")
        c["vis"] = own
        check_outputs(c, rr, sets, label)
        for b in range(B):
            private = rr["res"][b, 0, :, :][torch.arange(rr["res"].shape[-1], device=DEV)[None] < rr["nnz"][b, 0][:, None]]
            assert bool((private >= n).any()), f"request {b} sampled none of its spilled keys"
            c["win_k"][b] = torch.cat([c["win_k"][b], (c["k_new"][b, 0] - avg_of(c, b))[:, None]], dim=1)
            c["win_v"][b] = torch.cat([c["win_v"][b], c["v_new"][b, 0][:, None]], dim=1)

    private_step("after spill B8")
    ctx.fork(2, 5)   # request 5 continues request 2: its window and the private keys 2 sees
    vis[5] = list(vis[2])
    c["win_k"][5], c["win_v"][5] = c["win_k"][2].clone(), c["win_v"][2].clone()
    private_step("after spill and fork B8")


# ---- dense layers in shared-prefix mode --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 4])
@pytest.mark.parametrize("B", [8, 32])
@pytest.mark.parametrize("regime", ["R2", "R4"])
def test_dense_shared_prefix(cuda_lib, regime, B, T):
    """dense_tail_rows 16 over one 98 000-row prompt in the slot: each request kept a different number of rows of two earlier
    4-token steps (ragged tails); the step against fp64 over the prompt plus that request's own tail.  The dense kernel puts up
    to max(1, 32 / (T * G)) requests of one slot in a chunk (dense_slot_chunks), so these shapes form 1 (B = 8, T = 1), 4 or 16
    chunks; the library reports no chunk count, so this reading of the kernel is not asserted."""
    P = 98000
    c = make_dense_slots(regime, B, P, T, seed=seed_of("dense", regime, B, T))
    o, moved = check_dense_inputs(c)
    ctx = two_layer_context(4, 8, HQ, HKV, B, M_C2, GEN, synth.make_hash_func(d, 4, 8, seed=1), dict(out_f32=1),
                            alloc_dense_kv=True, max_query_tokens=4, num_contexts=1, dense_tail_rows=16)
    small = torch.randn((HKV, 64, d), generator=torch.Generator(device=DEV).manual_seed(1), device=DEV).bfloat16()
    ctx.attn_fill(1, 0, small, small, small.float().norm(dim=-1))
    ctx.lsh_build(1, 0, ctx.hash_keys(small))
    ctx.window_fill(1, 0, torch.zeros((HKV, d), dtype=torch.bfloat16, device=DEV), small, small)
    ctx.dense_fill(0, 0, c["dk"].contiguous(), c["dv"].contiguous(), P)
    for b in range(1, B):
        ctx.fork(0, b)
    for pq, pk, pv, drop in c["pre"]:
        ctx.plan(4)
        ctx.dense_decode_tokens(0, 4, pq, pk, pv)
        ctx.rewind(torch.tensor(drop, dtype=torch.int32, device=DEV))
    if T == 1:
        ctx.plan()
        out = ctx.dense_decode(0, c["q"][:, 0].contiguous(), c["k"][:, 0].contiguous(), c["v"][:, 0].contiguous())
    else:
        ctx.plan(T)
        out = ctx.dense_decode_tokens(0, T, c["q"], c["k"], c["v"])
    o32 = ctx.last_out_f32()
    assert ctx.error_flags() == 0
    worst = rel_rows(o32, o)
    label = f"dense B{B} T{T} {regime}"
    print(f"{label}: perturbations " + ", ".join(f"{k} {v:.2e}" for k, v in moved.items())
          + f"; largest relative head error {worst:.2e} ({worst / BAR:.1%} of the bar)")
    assert worst <= BAR, f"{label}: fp32 output differs from fp64 by {worst:.3e} relative"
    assert_rounded_half_up(out, o32, label)
