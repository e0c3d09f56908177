"""Attention kernels against an fp64 restatement on model-shaped inputs (`-m gpu`).

The other GPU files mostly check a path against a twin (T tokens against T single steps, a fork against a private copy) and
give the absolute check i.i.d. Gaussian inputs, on which the key mean is near zero, the window carries a few per cent of the
mass and the softmax is flat.  A kernel that forgot to centre the new key, dropped a window row or skipped a rescale passes
there.  The inputs here are shaped like a model's instead, one knob per regime:

  R1  key mean: keys = mu + noise with |mu| four times the per-key noise; the store and the window hold centred rows, the new
      tokens carry mu and the kernel must subtract avg_k itself;
  R2  sinks: the num_sink_tokens first window rows (and the new token) are aligned with every query of the group, so the window
      holds >= 90 % of the mass;
  R3  balanced: each query is scaled so that the window's share of the merged mass is 0.35 or 0.65;
  R4  large logits: queries x 16 (scores span >= 40 nats) and one dominant key, placed first or last in the store;
  R5  parallel keys: a few stored keys are exact bf16 multiples of a query, so cs rounds past 1 and the clamp is taken.

The restatement (`restate`) takes the sample set from collision counts over the GPU's own query codes (checked first against
an fp64 projection with the margin rule of test_simhash), clamps cos to [-1, 1], applies the LSH weight, attends the window
rows plus bf16(k_new - avg_k) under the causal / ancestor mask of the step, and merges the two halves by their base-2 LSEs,
all in fp64.  One exception: the weight 1 - (1-p)^(L-1) (Lp + 1 - p) is evaluated in the reference's fp32 order (as the C
oracle does), because for w <~ 1e-4 its fp32 cancellation is part of the reference's definition of the output, and a kernel
computing it in fp32 cannot be held to the fp64 value there.

Every generator checks, before any GPU call, that its inputs can tell a broken kernel from a correct one: a named perturbation
of the restatement (`SELF_CHECK`) must move the output by at least 10x the 1e-3 bar.
"""
import math
import zlib

import pytest
import torch

import oracle
from magicpig_b200 import synth
from tests.support.fp64 import BAR, SIMHASH_EPS, assert_1e3_f32, assert_rounded_half_up, rel_rows, sample_scores, sample_sets, \
    restate, softmax_state
from tests.support.library import DEV, NL, NS, Doc, d, two_layer_context
from tests.support.sparse_cases import TREE, check_case, check_dense, fill_case, make_case, make_dense, restate_dense

pytestmark = pytest.mark.gpu
GEN = 32


# ------------------------------------------------------------------------------------------------
# GPU side
# ------------------------------------------------------------------------------------------------
def check_codes(c, codes: torch.Tensor):
    """GPU query codes (B, T, Hq, L) against the fp64 projection of the query normalised as the reference does (bf16 norm, bf16
    quotient; oracle.simhash): a code may differ only where one of its K projections is within SIMHASH_EPS of zero
    (test_simhash's rule, no count allowance)."""
    ref, margin = oracle.simhash(c["q"].reshape(-1, d).contiguous(), c["hf"], c["K"], c["L"])
    bad = codes.reshape(ref.shape) != ref
    if bool(bad.any()):
        assert float(margin[bad].max()) < SIMHASH_EPS, f"{int(bad.sum())} query codes differ beyond rounding"


def check_lists(c, sets, nnz, res):
    B, T, Hq = nnz.shape
    for b in range(B):
        for t in range(T):
            for h in range(Hq):
                n_ = int(nnz[b, t, h])
                assert n_ == len(sets[b][t][h]), (b, t, h)
                assert torch.equal(res[b, t, h, :n_].long(), sets[b][t][h]), (b, t, h)


def sparse_ctx(c, impl=1, kreg=0, t_max=1, M=None, **opts):
    ctx = two_layer_context(c["K"], c["L"], c["Hq"], c["Hkv"], c["B"], M or c["n"] + 256, GEN, c["hf"],
                            dict(decode_impl=impl, fused_kreg=kreg, save_mask=1, out_f32=1, **opts), max_query_tokens=t_max)
    return fill_case(ctx, c)


def run_step(ctx, c, parents=None):
    """One step of c's T tokens (T = 1: plan + decode); returns readouts shaped (B, T, Hq, ...)."""
    B, T, Hq = c["q"].shape[:3]
    if T == 1:
        ctx.plan()
        out = ctx.decode(1, c["q"][:, 0].contiguous().to(DEV), c["k_new"][:, 0].contiguous().to(DEV),
                         c["v_new"][:, 0].contiguous().to(DEV))
    else:
        ctx.plan(T, parents=None if parents is None else torch.tensor(parents, dtype=torch.int32, device=DEV))
        out = ctx.decode_tokens(1, T, c["q"].to(DEV), c["k_new"].to(DEV), c["v_new"].to(DEV))
    nnz, res = ctx.last_probe(want_results=True)
    return dict(out=out.cpu().reshape(B, T, Hq, d), o32=ctx.last_out_f32().cpu().reshape(B, T, Hq, d),
                codes=ctx.last_codes().cpu().reshape(B, T, Hq, -1), nnz=nnz.cpu().reshape(B, T, Hq),
                res=res.cpu().reshape(B, T, Hq, -1))


def check_step(c, r, parents=None):
    """Codes, index lists and nnz against fp64; fp32 output within 1e-3 of the restatement; bf16 output = fp32 rounded once."""
    check_codes(c, r["codes"])
    sets = sample_sets(c, r["codes"])
    check_lists(c, sets, r["nnz"], r["res"])
    o, lse_s, _ = restate(c, r["codes"], parents=parents, sets=sets)
    assert_1e3_f32(r["o32"].reshape(-1, d), o.reshape(-1, d))
    assert_rounded_half_up(r["out"], r["o32"])
    return o, lse_s


SHAPES = [
    (1, 16, 4, 4096, 10, 150),     # clusters of 4
    (1, 4, 1, 1500, 8, 60),        # clusters of 8
    (1, 8, 1, 70000, 8, 40),       # two key segments
    (4, 32, 8, 2000, 8, 60),       # 128 heads, one CTA each
]
REGIMES = [("R1", "last"), ("R2", "last"), ("R3", "last"), ("R4", "first"), ("R4", "last"), ("R5", "last")]
_cases = {}


def case(regime, place, shape, T=1):
    key = (regime, place, shape, T)
    if key not in _cases:
        B, Hq, Hkv, n, K, L = shape
        c = make_case(regime, B, Hq, Hkv, n, K, L, seed=zlib.crc32(repr(key).encode()) % 10000, T=T, place=place)
        check_case(c)
        _cases[key] = c
    return _cases[key]


# ---- fused single-token decode, three-launch path, stand-alone gather kernel --------------------------------------------
@pytest.mark.parametrize("kreg", [0, 1])
@pytest.mark.parametrize("shape", SHAPES, ids=["c4", "c8", "seg2", "cta1"])
@pytest.mark.parametrize("regime,place", REGIMES, ids=[f"{r}{p[0]}" if r == "R4" else r for r, p in REGIMES])
def test_fused_decode_regimes(cuda_lib, regime, place, shape, kreg):
    c = case(regime, place, shape)
    ctx = sparse_ctx(c, impl=1, kreg=kreg)
    r = run_step(ctx, c)
    assert ctx.get_info("last_decode_fused") == 1
    check_step(c, r)


@pytest.mark.parametrize("tma", [0, 1])
@pytest.mark.parametrize("regime,place", REGIMES, ids=[f"{r}{p[0]}" if r == "R4" else r for r, p in REGIMES])
def test_three_launch_and_gather_regimes(cuda_lib, regime, place, tma):
    """decode_impl 0 (SimHash | probe | attend) and the stand-alone gather kernel (mpig_attention_wrapper), whose base-2 LSE
    (mve row 1) must match the sampled half's fp64 LSE."""
    c = case(regime, place, SHAPES[0])
    ctx = sparse_ctx(c, impl=0, attend_tma=tma)
    r = run_step(ctx, c)
    assert ctx.get_info("last_decode_fused") == 0
    _, lse_s = check_step(c, r)
    H = c["B"] * c["Hq"]
    res = torch.zeros((H, ctx.M), dtype=torch.int32)
    for i in range(H):
        res[i, : int(r["nnz"].reshape(-1)[i])] = r["res"].reshape(H, -1)[i, : int(r["nnz"].reshape(-1)[i])]
    out = torch.zeros((H, d), dtype=torch.bfloat16, device=DEV)
    mve = torch.zeros((2, H), dtype=torch.float32, device=DEV)
    q = c["q"][:, 0].reshape(H, d).contiguous()
    ctx.attention_wrapper(1, c["K"], c["L"], out, mve, q.to(DEV), q.float().norm(dim=-1).to(DEV), res.to(DEV),
                          r["nnz"].reshape(-1).contiguous().to(DEV))
    o32 = ctx.last_out_f32().cpu()
    sets = sample_sets(c, r["codes"])
    for i in range(H):
        b, h = divmod(i, c["Hq"])
        idx, st = sets[b][0][h], c["slots"][b]
        o_s, l_s = softmax_state(sample_scores(q[i], st["key"][h // c["G"], idx], st["kn"][h // c["G"], idx], c["K"], c["L"]),
                                 st["value"][h // c["G"], idx])
        assert_1e3_f32(o32[i][None], o_s[None])
        if l_s == -math.inf:
            assert float(mve[1, i]) == -math.inf
        else:
            assert abs(float(mve[1, i]) - l_s) <= BAR * max(1.0, abs(l_s)), (i, float(mve[1, i]), l_s)


# ---- T-token steps and a tree ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kreg", [0, 1])
@pytest.mark.parametrize("T,tree", [(3, False), (8, False), (8, True)], ids=["T3", "T8", "tree8"])
@pytest.mark.parametrize("regime", ["R1", "R2", "R3", "R4"])
def test_tokens_regimes(cuda_lib, regime, T, tree, kreg):
    """Every token of a step of T tokens (or node of an 8-node branching tree) directly against fp64, with the causal or
    ancestor mask over the step's rows."""
    B, Hq, Hkv, n, K, L = 2, 8, 2, 3000, 8, 60
    parents = [TREE] * B if tree else None
    c = make_case(regime, B, Hq, Hkv, n, K, L, seed=31 + T + 7 * tree, T=T, parents=parents)
    check_case(c, parents)
    ctx = sparse_ctx(c, kreg=kreg, t_max=T)
    check_step(c, run_step(ctx, c, parents), parents)


def test_decode_after_spill_r1(cuda_lib):
    """Under a large key mean, spilled window rows keep their centring: decode after spill_window against fp64 over the store
    as it now is (its keys, norms and the GPU's codes of them)."""
    B, Hq, Hkv, n, K, L = 2, 8, 2, 1500, 7, 40
    c = make_case("R1", B, Hq, Hkv, n, K, L, seed=5)
    check_case(c)
    ctx = sparse_ctx(c)
    g = torch.Generator().manual_seed(6)
    avg = torch.stack([st["avg"] for st in c["slots"]])
    win_k, win_v = torch.stack(c["win_k"]), torch.stack(c["win_v"])
    for _ in range(20):   # steps with new keys that carry the mean; the window gains their centred rows
        k_new = (torch.randn((B, Hkv, d), generator=g, dtype=torch.float64) + avg.double()).bfloat16()
        v_new = torch.randn((B, Hkv, d), generator=g).bfloat16()
        ctx.plan()
        ctx.decode(1, c["q"][:, 0].contiguous().to(DEV), k_new.to(DEV), v_new.to(DEV))
        win_k = torch.cat([win_k, (k_new - avg)[:, :, None]], dim=2)
        win_v = torch.cat([win_v, v_new[:, :, None]], dim=2)
    got = ctx.spill_window(NL)
    sp = int(got[0])
    assert got.tolist() == [sp] * B and sp == 20
    moved_k = win_k[:, :, NS:NS + sp]
    c["win_k"] = list(torch.cat([win_k[:, :, :NS], win_k[:, :, NS + sp:]], dim=2))
    c["win_v"] = list(torch.cat([win_v[:, :, :NS], win_v[:, :, NS + sp:]], dim=2))
    k_st, v_st, kn_st = (x.cpu() for x in ctx.read_cache(1))
    n2 = n + sp
    assert torch.equal(k_st[:, :, n:n2].view(torch.int16), moved_k.contiguous().view(torch.int16)), "spilled rows lost their centring"
    # the tables: the prompt's codes as built, the spilled rows' codes from the context's key hash (what the spill merged)
    c["n"] = n2
    for b, st in enumerate(c["slots"]):
        spilled_codes = ctx.hash_keys(k_st[b, :, n:n2].contiguous().to(DEV)).cpu()
        st.update(key=k_st[b, :, :n2].contiguous(), value=v_st[b, :, :n2].contiguous(), kn=kn_st[b, :, :n2].contiguous(),
                  kcodes=torch.cat([st["kcodes"], spilled_codes], dim=-1))
    # queries near the spilled keys, so that they are sampled
    q = (moved_k[:, :, 3:4].double().repeat_interleave(c["G"], dim=1).transpose(1, 2)
         + 0.25 * torch.randn((B, 1, Hq, d), generator=g, dtype=torch.float64)).bfloat16()
    c["q"] = q
    r = run_step(ctx, c)
    check_step(c, r)
    assert all(int((r["res"][b, 0, h, : r["nnz"][b, 0, h]] >= n).sum()) > 0 for b in range(B) for h in range(Hq))


# ---- dense layers ---------------------------------------------------------------------------------------------------------
def dense_ctx(B, Hq, Hkv, M, t_max=1, impl=1, **kw):
    # (K4 L8: tables unused)
    return two_layer_context(4, 8, Hq, Hkv, B, M, GEN, None, dict(dense_impl=impl, out_f32=1), alloc_dense_kv=True,
                             max_query_tokens=t_max, **kw)


def run_dense(ctx, c, parents=None):
    B, T, Hq = c["q"].shape[:3]
    if T == 1:
        ctx.plan()
        out = ctx.dense_decode(0, c["q"][:, 0].contiguous().to(DEV), c["k"][:, 0].contiguous().to(DEV), c["v"][:, 0].contiguous().to(DEV))
    else:
        ctx.plan(T, parents=None if parents is None else torch.tensor(parents, dtype=torch.int32, device=DEV))
        out = ctx.dense_decode_tokens(0, T, c["q"].to(DEV), c["k"].to(DEV), c["v"].to(DEV))
    o32 = ctx.last_out_f32().cpu().reshape(B, T, Hq, d)
    assert_rounded_half_up(out, o32)
    return o32


def fill_dense(ctx, c):
    for b in range(c["B"]):
        ctx.dense_fill(0, b, c["dk"][b].to(DEV).contiguous(), c["dv"][b].to(DEV).contiguous(), c["P"])


DENSE_P = [1, 31, 32, 33, 4095, 4097, 60000]


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("P", DENSE_P)
@pytest.mark.parametrize("regime,G", [("R2", None), ("R4", None), ("R2", 16), ("R4", 16), ("R2", 32), ("R4", 32)],
                         ids=["R2", "R4", "R2-G16", "R4-G16", "R2-G32", "R4-G32"])
def test_dense_single(cuda_lib, regime, G, P, impl):
    """Single-token dense decode (dense_impl 1: GQA-shared kernel, 0: generic gather) at tile edges, and at a P whose groups
    are split over several CTAs (level-2 merge).  G = 16 / 32: more query heads per kv-head than one packed m-tile holds, on
    one m-tile or two."""
    B, Hq, Hkv = (1, 8, 1) if P > 5000 else (2, 8, 2)
    if G:
        Hq = G * Hkv
    c = make_dense(regime, B, Hq, Hkv, P, 1, seed=P + 3, place="new" if P == 1 else ("first" if P % 2 else "last"))
    o = check_dense(c)
    ctx = dense_ctx(B, Hq, Hkv, P + 256, impl=impl)
    fill_dense(ctx, c)
    assert_1e3_f32(run_dense(ctx, c).reshape(-1, d), o.reshape(-1, d))


@pytest.mark.parametrize("tree", [False, True])
@pytest.mark.parametrize("G,T", [(4, 2), (4, 4), (4, 8)], ids=["TG8", "TG16", "TG32"])
@pytest.mark.parametrize("regime", ["R2", "R4"])
def test_dense_tokens(cuda_lib, regime, G, T, tree):
    B, Hkv, P = 2, 2, 777
    parents = [TREE[:T] if T < 8 else TREE] * B if tree else None
    c = make_dense(regime, B, G * Hkv, Hkv, P, T, seed=T + 50 * tree, place="last")
    o = check_dense(c, parents)
    ctx = dense_ctx(B, G * Hkv, Hkv, P + 256, t_max=T)
    fill_dense(ctx, c)
    assert_1e3_f32(run_dense(ctx, c, parents).reshape(-1, d), o.reshape(-1, d))


@pytest.mark.parametrize("T", [1, 4])
@pytest.mark.parametrize("regime", ["R2", "R4"])
def test_dense_slots(cuda_lib, regime, T):
    """Slot mode (dense_tail_rows > 0): the sink (R2) or the large logits' prompt lives in the shared prefix; in R4 the dominant
    key is appended to request 1's tail by its first step only.  Three steps; each request against fp64 over prompt + its tail."""
    B, Hq, Hkv, P = 4, 8, 2, 1000
    c = make_dense(regime, B, Hq, Hkv, P, T, seed=77 + T, place="new", one_prompt=True)
    if regime == "R4":
        c["k"][[0, 2, 3], -1] = c["k"][[0, 2, 3], 0]
    hf = synth.make_hash_func(d, 4, 8, seed=1)
    ctx = dense_ctx(B, Hq, Hkv, 2048, t_max=T, num_contexts=1, dense_tail_rows=64)
    ctx.set_hash_func(hf.to(DEV))
    doc = Doc(Hkv, 600, 4, 8, hf, seed=9, P_dense=P)
    doc.dk, doc.dv = c["dk"][0].clone(), c["dv"][0].clone()
    doc.fill_store(ctx, 0)
    doc.fill_request(ctx, 0)
    for b in range(1, B):
        ctx.fork(0, b)
    assert ctx.dense_tail_rows == 64
    g = torch.Generator().manual_seed(T)
    for step in range(3):
        o = check_dense(c) if step == 0 else restate_dense(c)
        assert_1e3_f32(run_dense(ctx, c).reshape(-1, d), o.reshape(-1, d))
        # the step's rows join every request's own rows; next step: new queries, keys and values of the same kind
        c["dk"], c["dv"] = torch.cat([c["dk"], c["k"]], dim=1), torch.cat([c["dv"], c["v"]], dim=1)
        fresh = torch.randn(c["k"].shape, generator=g, dtype=torch.float64)
        c["k"] = (0.25 * fresh + c["dk"][:, :1].double()).bfloat16() if regime == "R2" else fresh.bfloat16()
        c["v"] = torch.randn(c["v"].shape, generator=g).bfloat16()
        c["q"] = (c["q"].double() * (1.0 + 0.05 * torch.randn(c["q"].shape, generator=g, dtype=torch.float64))).bfloat16()


# ---- scale invariance and option paths ------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", [1, 0])
def test_scale_invariance(cuda_lib, impl):
    """q x 2^k: SimHash normalises q and a power of two scales it exactly, so codes, nnz and index lists are bitwise those of
    q; only the outputs move (and each stays within the bar of its own fp64 restatement)."""
    c = case("R1", "last", SHAPES[0])
    base = run_step(sparse_ctx(c, impl=impl), c)
    for k in (-3, 4):
        ck = dict(c, q=(c["q"].float() * 2.0 ** k).bfloat16())
        assert torch.equal(ck["q"].float(), c["q"].float() * 2.0 ** k)
        r = run_step(sparse_ctx(ck, impl=impl), ck)
        for key in ("codes", "nnz", "res"):
            assert torch.equal(r[key], base[key]), key
        assert not torch.equal(r["o32"], base["o32"])
        check_step(ck, r)


def _same(a, b, fp32_exact=True):
    for key in ("codes", "nnz", "res"):
        assert torch.equal(a[key], b[key]), key
    if fp32_exact:
        assert torch.equal(a["o32"], b["o32"])
    else:
        assert rel_rows(a["o32"], b["o32"]) <= 1e-5


@pytest.mark.parametrize("impl", [1, 0])
def test_issue_window_and_pdl(cuda_lib, impl):
    """fused_issue_win in {0, 1, 8, 32} and pdl_first in {0, 1}: bitwise the default's outputs, codes and lists."""
    c = case("R4", "last", SHAPES[2])
    base = run_step(sparse_ctx(c, impl=impl), c)
    check_step(c, base)
    for win in (0, 1, 8, 32):
        for pdl in (0, 1):
            _same(run_step(sparse_ctx(c, impl=impl, fused_issue_win=win, pdl_first=pdl), c), base)


def test_two_ctas_per_sm(cuda_lib, monkeypatch):
    """MPIG_CTA_PER_SM=2 (clusters of 512-thread CTAs): same index lists, fp32 within 1e-5, and within the bar of fp64."""
    c = case("R3", "last", SHAPES[0])
    base = run_step(sparse_ctx(c), c)
    monkeypatch.setenv("MPIG_CTA_PER_SM", "2")
    r = run_step(sparse_ctx(c), c)
    _same(r, base, fp32_exact=False)
    check_step(c, r)


def test_attend_ctas_warps(cuda_lib):
    """attend_ctas in {0, 1, 3} x attend_warps in {1, 5, 12} on the three-launch path: within 1e-5 of the default and 1e-3
    of fp64."""
    c = case("R2", "last", SHAPES[0])
    base = run_step(sparse_ctx(c, impl=0), c)
    check_step(c, base)
    for ctas in (0, 1, 3):
        for warps in (1, 5, 12):
            r = run_step(sparse_ctx(c, impl=0, attend_ctas=ctas, attend_warps=warps), c)
            _same(r, base, fp32_exact=False)
            check_step(c, r)
