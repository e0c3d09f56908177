"""The interval rule of tests/test_gpu_step_numerics.py, checked without a GPU.

Each aux kernel's fp32 arithmetic is emulated with numpy float32 in its real order (the GEMV's lane partition and shuffle
tree, the RMSNorm block reductions of add_rmsnorm and of the GEMV's fused prologue, SwiGLU on the rounded halves, RoPE) at
reduced but structurally identical shapes.  The emulations must pass the rule, and named mistakes must break it on at least
1 % of the elements, so a rule that has become too tight or too loose fails here first.  The fp64 step restatement is checked
the same way: each named perturbation moves a tiny model's logits by at least 10x a stand-in bar.
"""
import math

import numpy as np
import pytest
import torch

from magicpig_b200.llama_runner import rope_tables
from tests.support.fp64 import bf16_rne
from tests.support.step_rule import (Fp64Llama, U, assert_rule, gamma, gemv_ref, hull_ok, neighbours, prompt_kv, rmsnorm_ref,
                                     rope_cands, rule_ok, run_reference, run_rel_err, ss_roundings_add_rmsnorm,
                                     ss_roundings_prologue, swiglu_cands)

F32 = np.float32


# ------------------------------------------------------------------------------------------------
# float32 emulations of the kernels
# ------------------------------------------------------------------------------------------------
def bf16(a: np.ndarray) -> np.ndarray:
    """float32 -> bf16 (RNE) -> float32, the kernels' __float2bfloat16_rn."""
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).bfloat16().float().numpy()


def butterfly(a: np.ndarray) -> np.ndarray:
    """warp_sum over the last axis (32 lanes): xor shuffles 16, 8, 4, 2, 1 in fp32; every lane ends with the same value."""
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        a = (a + a[..., lane ^ o]).astype(F32)
    return a[..., 0]


def emu_gemv_acc(W: np.ndarray, x: np.ndarray, drop_last_step: bool = False) -> np.ndarray:
    """aux_gemv.cu's fp32 sums (before rounding): lane l of the warp owning row n adds w[k] x[k] for k = (s * 32 + l) * 8 + i,
    s over the K/256 steps, i over 8, in that order, then the shuffle tree.  W (N, K), x (rows, K) float32 bf16 values."""
    N, K = W.shape
    steps = K // 256
    Wr, xr = W.reshape(N, steps, 32, 8), x.reshape(x.shape[0], steps, 32, 8)
    acc = np.zeros((x.shape[0], N, 32), dtype=F32)
    for s in range(steps - drop_last_step):
        for i in range(8):
            acc = (acc + xr[:, None, s, :, i] * Wr[None, :, s, :, i]).astype(F32)   # the product of two bf16 is exact
    return butterfly(acc)


def silu_f32(g: np.ndarray, u: np.ndarray) -> np.ndarray:
    """(g / (1 + expf(-g))) * u in fp32 (expf correctly rounded here; overflow to inf below g = -88.72 as on the GPU)."""
    with np.errstate(over="ignore"):
        e = np.exp(-g.astype(F32)).astype(F32)
    return ((g / (F32(1) + e)).astype(F32) * u).astype(F32)


def emu_rmsnorm(h, delta, w, eps, threads: int, prologue: bool, over_h: bool = False, no_weight: bool = False):
    """add_rmsnorm_kernel (threads = 512: thread t owns chunks t and t + 512; the 16 warp sums by a second shuffle tree) or the
    GEMV's fused prologue (threads = 256: thread t owns chunks t, t + 256, ...; the 8 warp sums added in order).  Returns
    (stream, x) float32."""
    rows, H = h.shape
    v = h if delta is None else bf16(h + delta)
    vs = h if over_h else v
    nchunk = H // 8
    per = -(-nchunk // threads)
    pad = np.zeros((rows, per * threads * 8), dtype=F32)
    pad[:, :H] = vs
    V = pad.reshape(rows, per, threads, 8)
    ss = np.zeros((rows, threads), dtype=F32)
    for r in range(per):
        for i in range(8):
            ss = (ss + V[:, r, :, i] * V[:, r, :, i]).astype(F32)
    red = butterfly(ss.reshape(rows, threads // 32, 32))         # (rows, warps)
    if prologue:
        t = np.zeros(rows, dtype=F32)
        for wi in range(threads // 32):
            t = (t + red[:, wi]).astype(F32)
    else:
        t = butterfly(np.concatenate([red, np.zeros((rows, 32 - threads // 32), dtype=F32)], 1))
    inner = ((t / F32(H)).astype(F32) + F32(eps)).astype(F32)
    inv = (1.0 / np.sqrt(inner.astype(np.float64))).astype(F32)[:, None]
    ww = np.ones_like(w) if no_weight else w
    return v, bf16(((vs * inv).astype(F32) * ww).astype(F32))


def emu_rope(x: np.ndarray, cs: np.ndarray, sn: np.ndarray, cos_both: bool = False) -> np.ndarray:
    """rope_split_kernel / the GV_ROPE epilogue on bf16 x (..., 128): x1 c1 - x2 s1, x2 c2 + x1 s2 in fp32, rounded to bf16.
    cos_both: the mistake of using cos[t] / sin[t] for both halves."""
    x1, x2 = x[..., :64], x[..., 64:]
    c1, s1 = cs[..., :64], sn[..., :64]
    c2, s2 = (c1, s1) if cos_both else (cs[..., 64:], sn[..., 64:])
    return bf16(np.concatenate([(x1 * c1 - x2 * s1).astype(F32), (x2 * c2 + x1 * s2).astype(F32)], -1))


def T(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).double()


def outside(out, cands) -> float:
    """Share of elements the rule does not allow."""
    return float((~hull_ok(out, cands)).double().mean())


# ------------------------------------------------------------------------------------------------
# inputs (numpy, bf16 values)
# ------------------------------------------------------------------------------------------------
def rng(seed):
    return np.random.default_rng(seed)


def rows_with_outliers(r, rows, H, scale=1.0):
    h = r.standard_normal((rows, H)).astype(F32) * F32(scale)
    idx = r.integers(0, H, 6)
    h[0, idx] = (100.0 * 10.0 ** r.random(6) * np.where(r.random(6) < 0.5, -1, 1)).astype(F32)
    if rows >= 3:
        h[-1] = 0
    return bf16(h)


def mats(r, N, K):
    return bf16(r.standard_normal((N, K)).astype(F32) * F32(0.02))


# ------------------------------------------------------------------------------------------------
# the rule's pieces
# ------------------------------------------------------------------------------------------------
def test_bf16_rne_matches_the_fp32_conversion():
    """One rounding from fp64 agrees with torch's fp32 -> bf16 (RNE) wherever the value is an fp32; ties go to even."""
    r = rng(0)
    x = np.concatenate([r.standard_normal(100000) * 10.0 ** r.integers(-40, 38, 100000), [0.0, -0.0, 1e-40, -3e-39]]).astype(F32)
    got = bf16_rne(T(x))
    want = torch.from_numpy(x).bfloat16().double()
    assert torch.equal(got, want)
    ties = torch.tensor([1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, 256 + 1.0, 256 + 3.0], dtype=torch.float64)
    assert bf16_rne(ties).tolist() == [1.0, 1 + 4 * 2.0 ** -8, 256.0, 260.0]


def test_rule_allows_only_the_neighbours_of_a_midpoint():
    one, ulp = torch.tensor([1.0], dtype=torch.float64), 2.0 ** -7
    mid = one + ulp / 2
    assert bool(rule_ok(one, one + 0.3 * ulp, 1e-6)) and not bool(rule_ok(one + ulp, one + 0.3 * ulp, 1e-6))
    assert bool(rule_ok(one, mid + 1e-7, 1e-6)) and bool(rule_ok(one + ulp, mid - 1e-7, 1e-6))   # either neighbour
    assert not bool(rule_ok(one + 2 * ulp, mid, 1e-6)) and not bool(rule_ok(one - ulp, mid, 1e-6))
    assert not bool(rule_ok(torch.tensor([float("nan")]), one, 1.0))
    lo, hi = neighbours(mid, 1e-9)
    assert float(lo) == 1.0 and float(hi) == 1 + ulp


# ------------------------------------------------------------------------------------------------
# emulations pass the rule, named mistakes break it
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,N,K", [(1, 64, 256), (3, 40, 1280), (2, 33, 768), (8, 16, 2048)])
def test_gemv_emulation(rows, N, K):
    r = rng(rows * 100 + K)
    x, W = rows_with_outliers(r, rows, K), mats(r, 2 * N, K)
    ref, e = gemv_ref(T(W[:N]).bfloat16(), T(x))
    y = T(bf16(emu_gemv_acc(W[:N], x)))
    assert_rule("emu_gemv", y, [(ref, e)], ref)
    # SwiGLU on the rounded halves
    acc_g, acc_u = emu_gemv_acc(W[:N], x), emu_gemv_acc(W[N:], x)
    gr, eg = gemv_ref(T(W[:N]).bfloat16(), T(x))
    ur, eu = gemv_ref(T(W[N:]).bfloat16(), T(x))
    cands, canon = swiglu_cands(gr, eg, ur, eu)
    assert_rule("emu_swiglu", T(bf16(silu_f32(bf16(acc_g), bf16(acc_u)))), cands, canon)
    # mistakes: SwiGLU from the unrounded halves; the GEMV without its last k-step (K > 256)
    assert outside(T(bf16(silu_f32(acc_g, acc_u))), cands) >= 0.01
    if K > 256:
        assert outside(T(bf16(emu_gemv_acc(W[:N], x, drop_last_step=True))), [(ref, e)]) >= 0.01


@pytest.mark.parametrize("rows,H", [(1, 8), (4, 4104), (3, 8192), (5, 2048)])
def test_add_rmsnorm_emulation(rows, H):
    r = rng(H + rows)
    h, w = rows_with_outliers(r, rows, H), bf16((1 + 0.1 * r.standard_normal(H)).astype(F32))
    delta = bf16(r.standard_normal((rows, H)).astype(F32) * F32(0.5))
    if rows >= 3:
        delta[-1] = 0
    v, x = emu_rmsnorm(h, delta, w, 1e-5, 512, prologue=False)
    vr, xr, ex = rmsnorm_ref(T(h), T(delta), T(w), 1e-5, ss_roundings_add_rmsnorm())
    assert torch.equal(T(v), vr)
    assert_rule("emu_add_rmsnorm", T(x), [(xr, ex)], xr)
    _, x_h = emu_rmsnorm(h, delta, w, 1e-5, 512, prologue=False, over_h=True)
    _, x_w = emu_rmsnorm(h, delta, w, 1e-5, 512, prologue=False, no_weight=True)
    assert outside(T(x_h), [(xr, ex)]) >= 0.01          # RMSNorm over h instead of bf16(h + delta)
    assert outside(T(x_w), [(xr, ex)]) >= 0.01          # the weight ignored


@pytest.mark.parametrize("rows,K,N", [(1, 2048, 24), (3, 1280, 40), (8, 4096, 16)])
def test_norm_gemv_emulation(rows, K, N):
    """The fused prologue (its own reduction order) feeding the GEMV: the output must pass the rule with x's neighbours."""
    r = rng(K * 3 + rows)
    h, w = rows_with_outliers(r, rows, K), bf16((1 + 0.1 * r.standard_normal(K)).astype(F32))
    delta = bf16(r.standard_normal((rows, K)).astype(F32) * F32(0.5))
    W = mats(r, N, K)
    _, x = emu_rmsnorm(h, delta, w, 1e-5, 256, prologue=True)
    vr, xr, ex = rmsnorm_ref(T(h), T(delta), T(w), 1e-5, ss_roundings_prologue(K))
    assert_rule("emu_prologue", T(x), [(xr, ex)], xr)
    lo, hi = neighbours(xr, ex)
    ref, e = gemv_ref(T(W).bfloat16(), bf16_rne(xr), hi - lo)
    assert_rule("emu_norm_gemv", T(bf16(emu_gemv_acc(W, x))), [(ref, e)], ref)


def test_rope_emulation():
    r = rng(5)
    B, H = 6, 5
    qkv = bf16(r.standard_normal((B, H, 128)).astype(F32) * F32(3))
    cos, sin = bf16(r.standard_normal((64, 128)).astype(F32)), bf16(r.standard_normal((64, 128)).astype(F32))
    pos = r.integers(1, 64, B)
    cs, sn = cos[pos][:, None], sin[pos][:, None]
    cands, canon = rope_cands(T(qkv), 0.0, T(cs), T(sn))
    assert_rule("emu_rope", T(emu_rope(qkv, cs, sn)), cands, canon)
    assert outside(T(emu_rope(qkv, cs, sn, cos_both=True)), cands) >= 0.01             # cos[t] for both halves
    assert outside(T(emu_rope(qkv, cos[pos - 1][:, None], sin[pos - 1][:, None])), cands) >= 0.01   # pos - 1
    # the runner's tables: cos[t] == cos[t + 64], so only random tables can tell the halves apart
    rc, _ = rope_tables(500000.0, 128, 16, "cpu")
    assert torch.equal(rc[:, :64], rc[:, 64:])


def test_silu_emulation_overflow():
    """|g| up to 90: expf(-g) overflows below -88.72, the output is -0 * u, finite and inside the rule."""
    r = rng(9)
    g = bf16(np.concatenate([r.uniform(-90, 90, 4000), [-90.0, -89.0, -88.5, 90.0]]).astype(F32))
    u = bf16(r.standard_normal(g.shape).astype(F32) * F32(2))
    out = T(bf16(silu_f32(g, u)))
    assert bool(torch.isfinite(out).all())
    cands, canon = swiglu_cands(T(g), 0.0, T(u), 0.0)
    assert_rule("emu_silu", out, cands, canon)
    assert float(out[-4]) == 0.0 and float(canon[-4]) != 0.0      # the case the overflow term of the bound is for


# ------------------------------------------------------------------------------------------------
# the step restatement is sensitive
# ------------------------------------------------------------------------------------------------
STAND_IN_BAR = 5e-3


def tiny_model(hidden=512, inter=1024, Hq=4, Hkv=2, vocab=512, layers=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    d = 128

    def w(*s):
        return (torch.randn(s, generator=g) * (1.3 / math.sqrt(s[1]))).bfloat16().double()

    def ln():
        return (0.5 + torch.rand(hidden, generator=g)).bfloat16().double()

    cos, sin = rope_tables(500000.0, d, 1024, "cpu")
    return dict(Hq=Hq, Hkv=Hkv, eps=float(np.float32(1e-5)), embed=w(vocab, hidden), lm_head=w(vocab, hidden), norm=ln(),
                cos=cos.double(), sin=sin.double(),
                layers=[dict(ln1=ln(), wqkv=w((Hq + 2 * Hkv) * d, hidden), wo=w(hidden, Hq * d), ln2=ln(),
                             w_gate_up=w(2 * inter, hidden), w_down=w(hidden, inter)) for _ in range(layers)])


@pytest.mark.parametrize("perturb", Fp64Llama.PERTURBATIONS)
def test_step_restatement_is_sensitive(perturb):
    m = tiny_model()
    g = torch.Generator().manual_seed(1)
    B, P, steps = 2, 6, 4
    prompts = [[prompt_kv(g, P, 2) for _ in range(2)] for _ in range(B)]
    start = [P - 1, P - 1 + 150]
    ids = torch.randint(0, 512, (steps, B), generator=g).tolist()
    ref = run_reference(m, prompts, start, ids)
    bad = run_reference(m, prompts, start, ids, perturb)
    moved = run_rel_err(bad, ref)
    assert moved >= 10 * STAND_IN_BAR, moved


def test_bound_constants():
    """The bounds are a few hundred fp32 ulps at the model's shapes: far below a bf16 half-ulp (2^-9)."""
    assert gamma(14336 // 32 + 5) < 2.8e-5
    assert 0.5 * gamma(ss_roundings_add_rmsnorm() + 2) + 6 * U < 2 ** -9 / 1000
