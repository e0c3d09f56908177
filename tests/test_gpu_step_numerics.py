"""The decode step's GEMV, RMSNorm, RoPE and SwiGLU kernels (include/magicpig_b200_aux.h) against an fp64 restatement, and
the runner's whole step against an fp64 Llama (`-m gpu`).

The restatement rounds to bf16 (round to nearest even) exactly where the kernels' comments say they do:
  residual stream  bf16(h + delta);
  RMSNorm          mean of squares over the rounded stream, x = bf16(v * inv * w) rounded once (add_rmsnorm and the fused
                   prologue of the GEMV alike);
  GEMV             y = bf16(sum w_i x_i);
  SwiGLU           silu of the bf16-rounded gate and up, one rounding;
  RoPE             rotate-half on the bf16-rounded projection with the table's bf16 cos[p, t], sin[p, t], cos[p, t + 64],
                   sin[p, t + 64], one rounding;  v copied.

The interval rule: an output element must equal bf16(ref), except where ref lies within the kernel's fp32 error bound e of a
bf16 rounding midpoint; there it may be the other neighbour.  In general: the element must be the bf16 rounding of some value
in [ref - e, ref + e], and nothing else.  e is a worst-case bound of the kernel's own fp32 arithmetic (functions *_bound
below), never a count of tolerated mismatches.  Where a kernel rounds an intermediate the test cannot see (the GEMV output
before SwiGLU or RoPE, the normalised x inside the fused prologue), each neighbour that intermediate may take is allowed.
tests/test_step_numerics_cpu.py checks on a CPU that an emulation of each kernel's fp32 arithmetic in its real order passes
this rule and that named mistakes break it.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24                 # fp32 unit roundoff
TINY = 2.0 ** -149             # fp32 subnormal step: absolute floor of every bound
MPIG_EINVAL, MPIG_EUNSUPPORTED = -1, -5
OFF_MARGIN = {}                # kernel -> largest number of elements seen per call that differ from bf16(ref) inside the rule


# ------------------------------------------------------------------------------------------------
# bf16 rounding and the interval rule (device-agnostic torch, fp64)
# ------------------------------------------------------------------------------------------------
def bf16_rne(x: torch.Tensor) -> torch.Tensor:
    """fp64 -> the nearest bf16 value (ties to even), as fp64, in ONE rounding (no detour through fp32).  bf16 keeps 8
    significant bits; its subnormals are spaced 2^-133."""
    x = x.double()
    _, e = torch.frexp(x)
    ulp = torch.ldexp(torch.ones_like(x), (e - 8).clamp(min=-133))
    return torch.round(x / ulp) * ulp      # torch.round: half to even


def gamma(n: int) -> float:
    """Relative bound of n successive fp32 roundings."""
    return n * U / (1 - n * U)


def neighbours(ref: torch.Tensor, e) -> tuple:
    """The bf16 values an intermediate rounded from ref with fp32 error up to e may take: (lower, upper) (equal off a
    midpoint)."""
    return bf16_rne(ref - e), bf16_rne(ref + e)


def rule_ok(out: torch.Tensor, ref: torch.Tensor, e) -> torch.Tensor:
    """Elementwise: out is the bf16 rounding of some value in [ref - e, ref + e]."""
    lo, hi = neighbours(ref, e)
    o = out.double()
    return torch.isfinite(o) & (o >= lo) & (o <= hi)


def hull_ok(out: torch.Tensor, cands) -> torch.Tensor:
    """Elementwise: out lies between the smallest and the largest bf16 value the candidates (ref, e) allow.  The candidates
    are the corners of the range an output takes while an unseen rounded intermediate moves between its extreme values."""
    lo = hi = None
    for ref, e in cands:
        a, b = neighbours(ref, e)
        lo = a if lo is None else torch.minimum(lo, a)
        hi = b if hi is None else torch.maximum(hi, b)
    o = out.double()
    return torch.isfinite(o) & (o >= lo) & (o <= hi)


def assert_rule(name: str, out: torch.Tensor, cands, canon: torch.Tensor) -> int:
    """out must satisfy the rule over the hull of cands (hull_ok).  canon: the restatement with every intermediate rounded to
    nearest.  Returns the number of elements != bf16(canon)."""
    ok = hull_ok(out, cands)
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        i = tuple(bad[0].tolist())
        lo = min(float(bf16_rne(r - e)[i]) for r, e in cands)
        hi = max(float(bf16_rne(r + e)[i]) for r, e in cands)
        raise AssertionError(f"{name}: {len(bad)} of {out.numel()} elements outside the rule; first at {i}: got {float(out[i])!r}, "
                             f"bf16(ref) {float(bf16_rne(canon)[i])!r}, ref {float(canon[i])!r}, allowed [{lo!r}, {hi!r}]")
    off = int((out.double() != bf16_rne(canon)).sum())
    OFF_MARGIN[name] = max(OFF_MARGIN.get(name, 0), off)
    return off


# ------------------------------------------------------------------------------------------------
# fp64 restatements with the kernels' fp32 error bounds
# ------------------------------------------------------------------------------------------------
def gemv_bound(K: int, absum: torch.Tensor) -> torch.Tensor:
    """fp32 accumulation of aux_gemv.cu: each lane runs one FMA chain over K/256 steps x 8 elements (bf16 x bf16 products are
    exact in fp32), then a 5-level shuffle tree: at most K/32 + 5 roundings of partial sums bounded by sum |w_i x_i|."""
    return gamma(K // 32 + 5) * absum + TINY


def gemv_ref(W: torch.Tensor, x: torch.Tensor, spread: torch.Tensor | None = None):
    """y = x . W^T in fp64 and its bound.  W (N, K) bf16; x (rows, K) fp64 (bf16 values).  spread (rows, K): how far the
    kernel's own x may be from x (a neighbour of a rounded intermediate); it widens the bound by sum |w_i| spread_i."""
    K = W.shape[1]
    ax = x.abs() if spread is None else x.abs() + spread
    refs, errs = [], []
    for n0 in range(0, W.shape[0], 4096):
        w = W[n0:n0 + 4096].double()
        wa = w.abs()
        refs.append(x @ w.t())
        e = gemv_bound(K, ax @ wa.t())
        if spread is not None:
            e = e + spread @ wa.t()
        errs.append(e)
        del w, wa
    return torch.cat(refs, 1), torch.cat(errs, 1)


def ss_roundings_add_rmsnorm() -> int:
    """add_rmsnorm_kernel: <= 16 squares per thread (two chunks of 8), a warp shuffle tree (5), the 16 warp sums by a second
    shuffle tree (5)."""
    return 16 + 5 + 5


def ss_roundings_prologue(K: int) -> int:
    """The GEMV's fused prologue: K/256 squares per thread (256 threads, chunks of 8), a shuffle tree (5), 8 warp sums added
    in order (8)."""
    return K // 256 + 5 + 8


def rmsnorm_ref(h: torch.Tensor, delta, w: torch.Tensor, eps: float, n_ss: int):
    """(stream, x_ref, e): stream = bf16(h + delta) (exact), x_ref = stream * rsqrt(mean(stream^2) + eps) * w in fp64.
    Bound: the sum of squares carries n_ss roundings (the squares of bf16 values are exact in fp32), the division by hidden and
    the + eps one each: half of gamma(n_ss + 2) through the square root; rsqrtf is within 2 ulp (4u); v * inv * w adds two
    roundings."""
    v = h.double() if delta is None else bf16_rne(h.double() + delta.double())
    eps32 = float(np.float32(eps))
    inv = 1.0 / torch.sqrt((v * v).mean(-1, keepdim=True) + eps32)
    x = v * inv * w.double()
    rel = (0.5 * gamma(n_ss + 2) + 6 * U) * 1.001
    return v, x, rel * x.abs() + TINY


def silu(g: torch.Tensor) -> torch.Tensor:
    return g / (1.0 + torch.exp(-g))


G_STAR = -1.2784645427610738   # silu's minimum: silu is decreasing below it, increasing above


def silu_bound(val: torch.Tensor, g_lo: torch.Tensor, g_hi: torch.Tensor) -> torch.Tensor:
    """fp32 error of (g / (1 + __expf(-g))) * u = val for g in [g_lo, g_hi]: __expf is within 2 + floor(1.173 |g|) ulp (CUDA
    programming guide, intrinsic functions), then 1 + E, the division and the multiply round once each.  Below g = -88.72
    __expf overflows to inf and the kernels return -0 * u; the true value is below 90 e^-88.72 |u| ~ 3e-37 |u| there, so for
    g < -88 the bound also covers the distance to 0."""
    gmax = torch.maximum(g_lo.abs(), g_hi.abs())
    rel = ((3 + 1.2 * gmax) * 2.0 ** -23 + 3 * U) * 1.01
    return rel * val.abs() + torch.where(g_lo < -88.0, 1.01 * val.abs(), torch.zeros_like(val)) + TINY


def swiglu_cands(g_ref, e_g, u_ref, e_u):
    """Candidates (corners) for out = bf16(silu(bf16(g)) * bf16(u)) when g and u are rounded inside the kernel from ref +- e:
    g ranges over [g_lo, g_hi] and u over [u_lo, u_hi] (their extreme bf16 values); silu over the g range is bounded by its
    ends and, if inside, its minimum; the product of the two ranges by its four corners."""
    g_lo, g_hi = neighbours(g_ref, e_g)
    u_lo, u_hi = neighbours(u_ref, e_u)
    s_lo, s_hi = silu(g_lo), silu(g_hi)
    s_min = torch.minimum(s_lo, s_hi)
    s_min = torch.where((g_lo < G_STAR) & (g_hi > G_STAR), torch.full_like(s_min, float(silu(torch.tensor(G_STAR)))), s_min)
    s_max = torch.maximum(s_lo, s_hi)
    cands = []
    for s in (s_min, s_max):
        for u in (u_lo, u_hi):
            cands.append((s * u, silu_bound(s * u, g_lo, g_hi)))
    canon = silu(bf16_rne(g_ref)) * bf16_rne(u_ref)
    return cands, canon


def rope_cands(ref: torch.Tensor, e, cs: torch.Tensor, sn: torch.Tensor):
    """Candidates for the rotate-half RoPE of a projection rounded from ref +- e.  ref (..., 128) fp64; cs, sn (..., 128) the
    table rows (bf16 values, broadcast over heads).  x1 c1 - x2 s1 and x2 c2 + x1 s2: the products of bf16 values are exact in
    fp32, so the kernel rounds once in fp32 (u) and once to bf16."""
    lo, hi = neighbours(ref, e)
    c1, s1, c2, s2 = cs[..., :64], sn[..., :64], cs[..., 64:], sn[..., 64:]
    cands = []
    for a, b in ((lo, lo), (lo, hi), (hi, lo), (hi, hi)):
        x1, x2 = a[..., :64], b[..., 64:]
        o = torch.cat([x1 * c1 - x2 * s1, x2 * c2 + x1 * s2], -1)
        cands.append((o, U * o.abs() + TINY))
    r = bf16_rne(ref)
    canon = torch.cat([r[..., :64] * c1 - r[..., 64:] * s1, r[..., 64:] * c2 + r[..., :64] * s2], -1)
    return cands, canon


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------
def gen(seed: int) -> torch.Generator:
    return torch.Generator(device=DEV).manual_seed(seed)


def residual_rows(rows: int, hidden: int, g: torch.Generator, scale: float = 1.0) -> torch.Tensor:
    """(rows, hidden) bf16: N(0, scale); row 0 carries six outliers of 1e2..1e3 (late Llama layers have them); when rows >= 3
    the last row is zero."""
    h = torch.randn((rows, hidden), generator=g, device=DEV) * scale
    idx = torch.randint(0, hidden, (6,), generator=g, device=DEV)
    mag = 100.0 * 10.0 ** torch.rand((6,), generator=g, device=DEV)
    sign = torch.where(torch.rand((6,), generator=g, device=DEV) < 0.5, -1.0, 1.0)
    h[0, idx] = mag * sign
    if rows >= 3:
        h[-1] = 0
    return h.bfloat16()


def ln_weight(hidden: int, g: torch.Generator) -> torch.Tensor:
    return (1 + 0.1 * torch.randn((hidden,), generator=g, device=DEV)).bfloat16()


def weights(n: int, k: int, g: torch.Generator) -> torch.Tensor:
    return (torch.randn((n, k), generator=g, device=DEV) * 0.02).bfloat16()


def nan_like(shape) -> torch.Tensor:
    """An output buffer full of NaN: an element the kernel does not write fails the rule."""
    return torch.full(shape, float("nan"), dtype=torch.bfloat16, device=DEV)


POSITIONS = [0, 1, 97_999, 98_000 + 63, 499_999, 12_345, 64, 300_001]   # runner's tables: prompt start, bench context, C4 end


@pytest.fixture(scope="module")
def runner_tables():
    """The runner's RoPE tables at rope_theta = 500000, up to position 499 999."""
    from magicpig_b200.llama_runner import rope_tables
    return rope_tables(500000.0, 128, 500_000 + 8, DEV)


def tables_and_pos(kind: str, rows: int, runner_tables, g: torch.Generator):
    """('runner', the long-context positions) or ('random', N(0,1) tables whose two halves differ, random positions < 64)."""
    if kind == "runner":
        cos, sin = runner_tables
        pos = torch.tensor([POSITIONS[i % len(POSITIONS)] for i in range(rows)], dtype=torch.long, device=DEV)
    else:
        cos = torch.randn((64, 128), generator=g, device=DEV).bfloat16()
        sin = torch.randn((64, 128), generator=g, device=DEV).bfloat16()
        pos = torch.randint(0, 64, (rows,), generator=g, device=DEV, dtype=torch.long)
    return cos, sin, pos


# ------------------------------------------------------------------------------------------------
# the library
# ------------------------------------------------------------------------------------------------
def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture
def lib(cuda_lib):
    """The library with the programmatic-dependent-launch mask pinned to 0 (every runner construction sets it process-wide);
    the previous mask is restored afterwards."""
    old = cuda_lib.mpig_aux_set_pdl(0)
    yield cuda_lib
    cuda_lib.mpig_aux_set_pdl(old)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if OFF_MARGIN:
        print("\n[step numerics] largest count of elements != bf16(ref) inside the rule, per call:",
              ", ".join(f"{k} {v}" for k, v in sorted(OFF_MARGIN.items())))


def check(rc: int):
    from magicpig_b200 import _native as N
    N.check(rc)


# ------------------------------------------------------------------------------------------------
# 1. GEMV, plain and SwiGLU
# ------------------------------------------------------------------------------------------------
GEMV_CASES = (
    [(r, 6144, 4096, 0) for r in range(1, 9)]                                  # 8B q/k/v, every row count
    + [(r, 1000, 1280, 1) for r in range(1, 9)]                                # SwiGLU, every row count, 5 k-steps, ragged N
    + [(1, 4096, 4096, 0), (2, 4096, 4096, 0)]                                 # 8B o
    + [(1, 14336, 4096, 1), (2, 14336, 4096, 1), (8, 14336, 4096, 1)]          # 8B gate/up
    + [(1, 4096, 14336, 0), (2, 4096, 14336, 0), (7, 4096, 14336, 0)]          # 8B down; rows 7 x K 14336 = 196 KB of x
    + [(1, 10240, 8192, 0), (2, 10240, 8192, 0)]                               # 70B q/k/v
    + [(1, 28672, 8192, 1), (2, 28672, 8192, 1)]                               # 70B gate/up
    + [(1, 8192, 28672, 0), (3, 8192, 28672, 0)]                               # 70B down
    + [(1, 1280, 8192, 0), (2, 1280, 8192, 0)]                                 # 70B TP-8 rank q/k/v
    + [(1, 3584, 8192, 1), (2, 3584, 8192, 1), (1, 8192, 3584, 0), (2, 8192, 3584, 0)]   # 70B megatron TP-8 gate/up, down
    + [(3, 1, 256, 0), (5, 7, 768, 0), (4, 13, 1280, 1), (8, 33, 256, 1), (6, 1001, 768, 0)]   # ragged N
    + [(2, 2048, 256, 0), (3, 2048, 768, 1), (1, 2048, 1280, 0)]               # K of 1, 3 and 5 k-steps
    + [(8, 64, 12800, 0), (8, 40, 12800, 1)]                                   # rows 8 x K 12800 = exactly 200 KB
)


@pytest.mark.parametrize("rows,N,K,swiglu", GEMV_CASES)
def test_gemv(lib, rows, N, K, swiglu):
    g = gen(rows * 1009 + N * 7 + K + swiglu)
    x = residual_rows(rows, K, g)
    W = weights((2 if swiglu else 1) * N, K, g)
    y = nan_like((rows, N))
    check(lib.mpig_aux_gemv(P(W), P(x), P(y), rows, N, K, swiglu, stream()))
    torch.cuda.synchronize()
    if not swiglu:
        ref, e = gemv_ref(W, x.double())
        assert_rule("gemv", y, [(ref, e)], ref)
    else:
        gr, eg = gemv_ref(W[:N], x.double())
        ur, eu = gemv_ref(W[N:], x.double())
        cands, canon = swiglu_cands(gr, eg, ur, eu)
        assert_rule("gemv_swiglu", y, cands, canon)


def test_gemv_shared_memory_edge(lib):
    """rows * K * 2 <= 200 KB: rows 8 / K 13056 (204 KB) is refused before any launch and leaves y untouched; rows 8 / K 12800
    (exactly 200 KB) runs (test_gemv)."""
    g = gen(13056)
    x = residual_rows(8, 13056, g)
    W = weights(64, 13056, g)
    y = torch.randn((8, 64), generator=g, device=DEV).bfloat16()
    y0 = y.clone()
    for swiglu in (0, 1):
        assert lib.mpig_aux_gemv(P(W), P(x), P(y), 8, 32 if swiglu else 64, 13056, swiglu, stream()) == MPIG_EUNSUPPORTED
    torch.cuda.synchronize()
    assert torch.equal(y, y0)


# ------------------------------------------------------------------------------------------------
# 2. residual add + RMSNorm prologue fused into the GEMV
# ------------------------------------------------------------------------------------------------
NORM_GEMV_CASES = ([(r, hs, 1000, sw, dl) for r in range(1, 9) for hs in (4096, 8192) for sw in (0, 1) for dl in (True, False)]
                   + [(1, 4096, 14336, 1, True), (2, 4096, 14336, 1, True), (2, 8192, 28672, 1, True)])


def prologue_x(h, delta, lnw, eps, K):
    """The fused prologue's (stream, x canonical, spread): x is rounded inside the kernel, so each element may be either
    neighbour of its reference; spread = the distance between them (0 off a midpoint)."""
    v, xr, ex = rmsnorm_ref(h, delta, lnw, eps, ss_roundings_prologue(K))
    lo, hi = neighbours(xr, ex)
    return v, bf16_rne(xr), hi - lo


@pytest.mark.parametrize("rows,hs,N,swiglu,with_delta", NORM_GEMV_CASES)
def test_norm_gemv(lib, rows, hs, N, swiglu, with_delta):
    g = gen(rows * 31 + hs + N + 2 * swiglu + with_delta)
    h = residual_rows(rows, hs, g)
    delta = (torch.randn((rows, hs), generator=g, device=DEV) * 0.5).bfloat16() if with_delta else None
    if delta is not None and rows >= 3:
        delta[-1] = 0                                       # the zero row stays zero: x = 0, finite
    lnw = ln_weight(hs, g)
    W = weights((2 if swiglu else 1) * N, hs, g)
    h0 = h.clone()
    h_out, y = nan_like((rows, hs)), nan_like((rows, N))
    check(lib.mpig_aux_norm_gemv(P(W), P(h), P(delta), P(lnw), 1e-5, P(h_out), P(y), rows, N, hs, swiglu, stream()))
    torch.cuda.synchronize()
    v, xc, spread = prologue_x(h, delta, lnw, 1e-5, hs)
    assert torch.equal(h, h0)
    assert torch.equal(h_out.double(), v)                   # the residual stream: bitwise
    if not swiglu:
        ref, e = gemv_ref(W, xc, spread)
        assert_rule("norm_gemv", y, [(ref, e)], ref)
    else:
        gr, eg = gemv_ref(W[:N], xc, spread)
        ur, eu = gemv_ref(W[N:], xc, spread)
        cands, canon = swiglu_cands(gr, eg, ur, eu)
        assert_rule("norm_gemv_swiglu", y, cands, canon)


# ------------------------------------------------------------------------------------------------
# 3. norm + q/k/v projection + RoPE
# ------------------------------------------------------------------------------------------------
HEADS = [(32, 8, 4096), (8, 1, 8192), (4, 4, 4096)]     # 8B layer, 70B TP-8 rank, GQA 1


def rope_qkv_checks(name, q, k, v, ref, e, cos, sin, pos, Hq, Hkv, v_exact=None):
    """q / k against the RoPE candidates of the projection ref (rows, Hq + 2 Hkv, 128) +- e, v against ref itself (or bitwise
    against v_exact)."""
    cs, sn = cos[pos].double()[:, None], sin[pos].double()[:, None]
    for out, sl, nm in ((q, slice(0, Hq), "q"), (k, slice(Hq, Hq + Hkv), "k")):
        cands, canon = rope_cands(ref[:, sl], e if not torch.is_tensor(e) else e[:, sl], cs, sn)
        assert_rule(f"{name}_{nm}", out, cands, canon)
    vr = ref[:, Hq + Hkv:]
    if v_exact is not None:
        assert torch.equal(v.double(), v_exact)
    else:
        assert_rule(f"{name}_v", v, [(vr, e[:, Hq + Hkv:])], vr)


@pytest.mark.parametrize("tables", ["runner", "random"])
@pytest.mark.parametrize("Hq,Hkv,hs", HEADS)
@pytest.mark.parametrize("rows", range(1, 9))
def test_norm_qkv_rope(lib, runner_tables, rows, Hq, Hkv, hs, tables):
    g = gen(rows * 131 + Hq * 7 + Hkv + hs + (tables == "random"))
    nqkv = (Hq + 2 * Hkv) * 128
    h = residual_rows(rows, hs, g)
    delta = (torch.randn((rows, hs), generator=g, device=DEV) * 0.5).bfloat16() if rows % 2 else None
    lnw = ln_weight(hs, g)
    W = weights(nqkv, hs, g)
    cos, sin, pos = tables_and_pos(tables, rows, runner_tables, g)
    h_out = nan_like((rows, hs))
    q, k, v = nan_like((rows, Hq, 128)), nan_like((rows, Hkv, 128)), nan_like((rows, Hkv, 128))
    check(lib.mpig_aux_norm_qkv_rope(P(W), P(h), P(delta), P(lnw), 1e-5, P(h_out), P(cos), P(sin), P(pos), P(q), P(k), P(v),
                                     rows, Hq, Hkv, hs, stream()))
    # the same prologue and per-row accumulation with the plain epilogue (the PRE, GV_PLAIN instantiation), then rope_split:
    # bitwise the same q / k / v (RoPE rounds products of bf16 values once, in any order)
    h_out2, qkv = nan_like((rows, hs)), nan_like((rows, nqkv))
    check(lib.mpig_aux_norm_gemv(P(W), P(h), P(delta), P(lnw), 1e-5, P(h_out2), P(qkv), rows, nqkv, hs, 0, stream()))
    q2, k2, v2 = nan_like((rows, Hq, 128)), nan_like((rows, Hkv, 128)), nan_like((rows, Hkv, 128))
    check(lib.mpig_aux_rope_split(P(qkv), P(cos), P(sin), P(pos), P(q2), P(k2), P(v2), rows, Hq, Hkv, stream()))
    torch.cuda.synchronize()
    v_ref, xc, spread = prologue_x(h, delta, lnw, 1e-5, hs)
    assert torch.equal(h_out.double(), v_ref) and torch.equal(h_out2, h_out)
    ref, e = gemv_ref(W, xc, spread)
    ref, e = ref.reshape(rows, Hq + 2 * Hkv, 128), e.reshape(rows, Hq + 2 * Hkv, 128)
    rope_qkv_checks("norm_qkv_rope", q, k, v, ref, e, cos, sin, pos, Hq, Hkv)
    assert torch.equal(v, qkv.reshape(rows, -1, 128)[:, Hq + Hkv:])      # v is the projection, copied
    assert torch.equal(q, q2) and torch.equal(k, k2) and torch.equal(v, v2)


# ------------------------------------------------------------------------------------------------
# 4. add_rmsnorm, rope_split, silu_mul
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hidden", [8, 4096, 4104, 8192])
def test_add_rmsnorm(lib, hidden):
    """rows 1..32 (shared-context batches reach B = 32), with and without delta; 4104 leaves thread 0 alone in the second
    chunk, 8192 fills both chunks of every thread."""
    g = gen(hidden)
    n_ss = ss_roundings_add_rmsnorm()
    for rows in range(1, 33):
        h = residual_rows(rows, hidden, g)
        lnw = ln_weight(hidden, g)
        for with_delta in (True, False):
            delta = (torch.randn((rows, hidden), generator=g, device=DEV) * 0.5).bfloat16() if with_delta else None
            if delta is not None and rows >= 3:
                delta[-1] = 0
            hh, x = h.clone(), nan_like((rows, hidden))
            check(lib.mpig_aux_add_rmsnorm(P(hh), P(delta), P(lnw), 1e-5, P(x), rows, hidden, stream()))
            torch.cuda.synchronize()
            v, xr, ex = rmsnorm_ref(h, delta, lnw, 1e-5, n_ss)
            assert torch.equal(hh.double(), v), (rows, with_delta)        # in-place residual stream: bitwise
            assert_rule("add_rmsnorm", x, [(xr, ex)], xr)


def test_add_rmsnorm_refuses_wide_rows(lib):
    """hidden 8200 > 16 x 512: refused before any launch, nothing written."""
    g = gen(8200)
    h = torch.randn((2, 8200), generator=g, device=DEV).bfloat16()
    w, x = ln_weight(8200, g), torch.zeros((2, 8200), dtype=torch.bfloat16, device=DEV)
    h0 = h.clone()
    assert lib.mpig_aux_add_rmsnorm(P(h), P(h), P(w), 1e-5, P(x), 2, 8200, stream()) == MPIG_EINVAL
    torch.cuda.synchronize()
    assert torch.equal(h, h0) and not bool(x.any())


@pytest.mark.parametrize("tables", ["runner", "random"])
@pytest.mark.parametrize("Hq,Hkv", [(32, 8), (8, 1), (4, 4)])
@pytest.mark.parametrize("B", [1, 5, 32])
def test_rope_split(lib, runner_tables, B, Hq, Hkv, tables):
    g = gen(B * 17 + Hq + Hkv + (tables == "random"))
    nh = Hq + 2 * Hkv
    qkv = (torch.randn((B, nh * 128), generator=g, device=DEV) * (1 + 10 * torch.rand((B, 1), generator=g, device=DEV))).bfloat16()
    cos, sin, pos = tables_and_pos(tables, B, runner_tables, g)
    q, k, v = nan_like((B, Hq, 128)), nan_like((B, Hkv, 128)), nan_like((B, Hkv, 128))
    check(lib.mpig_aux_rope_split(P(qkv), P(cos), P(sin), P(pos), P(q), P(k), P(v), B, Hq, Hkv, stream()))
    torch.cuda.synchronize()
    ref = qkv.double().reshape(B, nh, 128)
    rope_qkv_checks("rope_split", q, k, v, ref, 0.0, cos, sin, pos, Hq, Hkv, v_exact=ref[:, Hq + Hkv:])


@pytest.mark.parametrize("rows,inter", [(160, 14336), (3, 8)])
def test_silu_mul(lib, rows, inter):
    """160 x 14336 runs the grid-stride loop twice on 132 SMs (8 blocks of 256 threads per SM, 8 elements per thread).  Half
    the rows have gates uniform in [-90, 90], where __expf(-g) overflows; those outputs stay finite and inside the rule."""
    g = gen(rows + inter)
    gate = torch.randn((rows, inter), generator=g, device=DEV) * 3
    wide = torch.rand((rows, inter), generator=g, device=DEV) * 180 - 90
    gate = torch.where((torch.arange(rows, device=DEV) % 2 == 1)[:, None], wide, gate)
    gate[0, :4] = torch.tensor([-90.0, 90.0, -88.5, -89.0], device=DEV)
    up = torch.randn((rows, inter), generator=g, device=DEV) * 2
    gu = torch.cat([gate, up], 1).bfloat16()
    out = nan_like((rows, inter))
    check(lib.mpig_aux_silu_mul(P(gu), P(out), rows, inter, stream()))
    torch.cuda.synchronize()
    cands, canon = swiglu_cands(gu[:, :inter].double(), 0.0, gu[:, inter:].double(), 0.0)
    assert_rule("silu_mul", out, cands, canon)


# ------------------------------------------------------------------------------------------------
# 5. programmatic dependent launch: the same bits under every mask
# ------------------------------------------------------------------------------------------------
def test_pdl_masks_bitwise(lib, runner_tables):
    """Each GEMV entry under mpig_aux_set_pdl(0|1|2|3), every call right behind the kernel that writes its input (bit 1 makes
    the plain GEMV wait on that producer), outputs bitwise equal across masks and inside the rule."""
    g = gen(77)
    rows, hs, Hq, Hkv, it = 2, 4096, 32, 8, 14336
    nqkv = (Hq + 2 * Hkv) * 128
    x_src, h_src = residual_rows(rows, hs, g), residual_rows(rows, hs, g)
    delta = (torch.randn((rows, hs), generator=g, device=DEV) * 0.5).bfloat16()
    lnw = ln_weight(hs, g)
    wo, wqkv, wgu = weights(hs, Hq * 128, g), weights(nqkv, hs, g), weights(2 * it, hs, g)
    cos, sin, pos = tables_and_pos("runner", rows, runner_tables, g)
    results = {}
    for mask in (0, 1, 2, 3):
        lib.mpig_aux_set_pdl(mask)
        x = torch.empty_like(x_src); x.copy_(x_src)                          # the producer
        y = nan_like((rows, hs))
        check(lib.mpig_aux_gemv(P(wo), P(x), P(y), rows, hs, Hq * 128, 0, stream()))
        x.copy_(x_src)
        act = nan_like((rows, it))
        check(lib.mpig_aux_gemv(P(wgu), P(x), P(act), rows, it, hs, 1, stream()))
        h = torch.empty_like(h_src); h.copy_(h_src)
        h2, q, k, v = nan_like((rows, hs)), nan_like((rows, Hq, 128)), nan_like((rows, Hkv, 128)), nan_like((rows, Hkv, 128))
        check(lib.mpig_aux_norm_qkv_rope(P(wqkv), P(h), P(delta), P(lnw), 1e-5, P(h2), P(cos), P(sin), P(pos), P(q), P(k), P(v),
                                         rows, Hq, Hkv, hs, stream()))
        h3, act2 = nan_like((rows, hs)), nan_like((rows, it))
        check(lib.mpig_aux_norm_gemv(P(wgu), P(h2), P(y), P(lnw), 1e-5, P(h3), P(act2), rows, it, hs, 1, stream()))
        h4, z = nan_like((rows, hs)), nan_like((rows, hs))
        check(lib.mpig_aux_norm_gemv(P(wo), P(h3), None, P(lnw), 1e-5, P(h4), P(z), rows, hs, hs, 0, stream()))
        torch.cuda.synchronize()
        results[mask] = [y, act, h2, q, k, v, h3, act2, h4, z]
    lib.mpig_aux_set_pdl(0)
    for mask in (1, 2, 3):
        for i, (a, b) in enumerate(zip(results[0], results[mask])):
            assert torch.equal(a, b), (mask, i)
    y, act = results[0][0], results[0][1]
    ref, e = gemv_ref(wo, x_src.double())
    assert_rule("gemv", y, [(ref, e)], ref)
    gr, eg = gemv_ref(wgu[:it], x_src.double())
    ur, eu = gemv_ref(wgu[it:], x_src.double())
    cands, canon = swiglu_cands(gr, eg, ur, eu)
    assert_rule("gemv_swiglu", act, cands, canon)


# ------------------------------------------------------------------------------------------------
# 6. the runner's step against an fp64 Llama
# ------------------------------------------------------------------------------------------------
class Fp64Llama:
    """An independent fp64 Llama decode over given weights: embedding, RMSNorm * w, q/k/v, rotate-half RoPE at the absolute
    position (the bf16 tables), GQA attention (query head h on KV head h // G) over the prompt and every generated token,
    o-projection and residual, SwiGLU MLP and residual, final norm, lm_head.  Everything stays fp64 except the generated
    tokens' K and V, which are kept rounded to bf16 as the server stores them.

    perturb names a deliberate mistake: 'rope_pos_minus_1', 'kv_head_mod' (query head h reads KV head h % Hkv), 'drop_newest'
    (the token being decoded does not attend to itself), 'no_ln_weight', 'swap_gate_up'."""

    PERTURBATIONS = ("rope_pos_minus_1", "kv_head_mod", "drop_newest", "no_ln_weight", "swap_gate_up")

    def __init__(self, m: dict, B: int, perturb: str | None = None):
        self.m, self.B, self.perturb = m, B, perturb
        self.Hq, self.Hkv, self.d, self.eps = m["Hq"], m["Hkv"], 128, m["eps"]
        self.kc = [[None] * len(m["layers"]) for _ in range(B)]
        self.vc = [[None] * len(m["layers"]) for _ in range(B)]

    def prefill(self, b: int, layer: int, k: torch.Tensor, v: torch.Tensor):
        self.kc[b][layer], self.vc[b][layer] = k.double(), v.double()      # (P, Hkv, d)

    def _norm(self, x, w):
        x = x / torch.sqrt((x * x).mean(-1, keepdim=True) + self.eps)
        return x if self.perturb == "no_ln_weight" else x * w

    def _rope(self, x, pos):
        p = pos - 1 if self.perturb == "rope_pos_minus_1" else pos
        c, s = self.m["cos"][p], self.m["sin"][p]
        return x * c + torch.cat([-x[..., 64:], x[..., :64]], -1) * s

    def step(self, ids, pos) -> torch.Tensor:
        """ids, pos: host int lists (B,).  Returns logits (B, vocab) fp64."""
        m, Hq, Hkv, d = self.m, self.Hq, self.Hkv, self.d
        G = Hq // Hkv
        heads = torch.arange(Hq, device=m["embed"].device)
        kvh = heads % Hkv if self.perturb == "kv_head_mod" else heads // G
        out = []
        for b in range(self.B):
            h = m["embed"][ids[b]]
            for li, lw in enumerate(m["layers"]):
                qkv = lw["wqkv"] @ self._norm(h, lw["ln1"])
                q = self._rope(qkv[:Hq * d].reshape(Hq, d), pos[b])
                k = self._rope(qkv[Hq * d:(Hq + Hkv) * d].reshape(Hkv, d), pos[b])
                v = qkv[(Hq + Hkv) * d:].reshape(Hkv, d)
                K = self.kc[b][li] = torch.cat([self.kc[b][li], bf16_rne(k)[None]], 0)
                V = self.vc[b][li] = torch.cat([self.vc[b][li], bf16_rne(v)[None]], 0)
                if self.perturb == "drop_newest":
                    K, V = K[:-1], V[:-1]
                Ks, Vs = K[:, kvh], V[:, kvh]                                   # (n, Hq, d)
                p = torch.softmax(torch.einsum("nhd,hd->hn", Ks, q) / math.sqrt(d), -1)
                a = torch.einsum("hn,nhd->hd", p, Vs).reshape(Hq * d)
                h = h + lw["wo"] @ a
                gu = lw["w_gate_up"] @ self._norm(h, lw["ln2"])
                it = gu.shape[0] // 2
                gt, up = (gu[it:], gu[:it]) if self.perturb == "swap_gate_up" else (gu[:it], gu[it:])
                h = h + lw["w_down"] @ (gt / (1 + torch.exp(-gt)) * up)
            out.append(m["lm_head"] @ self._norm(h, m["norm"]))
        return torch.stack(out)


def rel_err(a: torch.Tensor, ref: torch.Tensor) -> float:
    return float((a.double() - ref).norm() / ref.norm())


STEP_SHAPE = dict(layers=2, hidden=4096, inter=14336, Hq=32, Hkv=8, vocab=4096)
STEP_P, STEP_STEPS, STEP_SEED = 6, 4, 5
# Bar on the relative logits error ||logits - ref|| / ||ref|| of each step and request.  Largest value measured over every
# route below on an H100 80GB HBM3 (700 W power limit): 1.36e-2 (eager, B = 2; the GEMV, GEMM and graph routes 1.13e-2 to
# 1.24e-2), all of it the bf16 rounding of the step's activations and residual stream.  The bar is about 4x that.
STEP_BAR = 5e-2


def make_runner(B: int, fused: bool):
    from magicpig_b200.llama_runner import LlamaDecodeRunner, LlamaShape
    s = STEP_SHAPE
    shape = LlamaShape("Llama-3.1-8B layer", s["layers"], s["hidden"], s["inter"], s["Hq"], s["Hkv"], s["vocab"], 500000.0, 1e-5)
    r = LlamaDecodeRunner(shape, 8, 40, B, 512, device=DEV, seed=STEP_SEED, generation_buffer=16,
                          dense_layers=tuple(range(s["layers"])), fused=fused)
    g = torch.Generator().manual_seed(11)                  # non-unit norm weights, the same for every route
    for lw in r.layers:
        lw["ln1"].copy_(0.5 + torch.rand(s["hidden"], generator=g))
        lw["ln2"].copy_(0.5 + torch.rand(s["hidden"], generator=g))
    r.norm.copy_(0.5 + torch.rand(s["hidden"], generator=g))
    return r


def prompt_kv(g: torch.Generator, P: int, Hkv: int):
    """(k, v) (P, Hkv, 128) bf16 of a prompt on which the step's attention matters: a short prompt, so the token being
    decoded carries a large share of the attention, and keys three times larger on the 8 highest-frequency RoPE pairs (dims
    0..7 and 64..71), so that the scores depend on the rotation of q."""
    scale = torch.ones(128)
    scale[0:8] = scale[64:72] = 3.0
    k = (torch.randn((P, Hkv, 128), generator=g) * scale).bfloat16()
    v = torch.randn((P, Hkv, 128), generator=g).bfloat16()
    return k, v


def prompt(b: int, layer: int):
    return prompt_kv(torch.Generator().manual_seed(1000 + 10 * b + layer), STEP_P, STEP_SHAPE["Hkv"])


def run_rel_err(got, ref) -> float:
    """Relative distance between the logits of two runs (every step and request)."""
    return rel_err(torch.stack(list(got)), torch.stack(list(ref)))


def start_pos(b: int) -> int:
    return STEP_P - 1 + 150 * b


def step_ids(B: int):
    g = torch.Generator().manual_seed(B)
    return torch.randint(0, STEP_SHAPE["vocab"], (STEP_STEPS, B), generator=g).tolist()


@pytest.fixture(scope="module")
def fp64_model(cuda_lib):
    """The runner's weights (seed STEP_SEED, the norm weights of make_runner) in fp64, with its RoPE tables."""
    r = make_runner(1, True)
    m = dict(Hq=STEP_SHAPE["Hq"], Hkv=STEP_SHAPE["Hkv"], eps=float(np.float32(r.shape.rms_norm_eps)),
             embed=r.embed.double(), lm_head=r.lm_head.double(), norm=r.norm.double(), cos=r.cos.double(), sin=r.sin.double(),
             layers=[{k: t.double() for k, t in lw.items()} for lw in r.layers])
    del r
    torch.cuda.empty_cache()
    return m


def run_reference(m, prompts, start, ids, perturb=None):
    """Logits of every step: prompts[b][layer] = (k, v) (P, Hkv, d), start[b] = the prompt's last position, ids[t][b]."""
    B = len(prompts)
    ref = Fp64Llama(m, B, perturb)
    for b in range(B):
        for li, (k, v) in enumerate(prompts[b]):
            ref.prefill(b, li, k, v)
    return [ref.step(ids[t], [start[b] + 1 + t for b in range(B)]) for t in range(len(ids))]


def reference_logits(m, B: int, ids, perturb=None):
    prompts = [[tuple(t.to(DEV) for t in prompt(b, li)) for li in range(STEP_SHAPE["layers"])] for b in range(B)]
    return run_reference(m, prompts, [start_pos(b) for b in range(B)], ids, perturb)


ROUTES = [("gemv", 1), ("gemv", 2), ("gemm", 3), ("eager", 2), ("graph", 1), ("graph", 3)]
STEP_ERRORS = {}


@pytest.mark.parametrize("route,B", ROUTES, ids=[f"{r}-B{b}" for r, b in ROUTES])
def test_runner_step_matches_fp64_model(lib, fp64_model, route, B):
    """Four steps of the runner against the fp64 model.  B <= 2 runs the GEMV with the fused prologues, B = 3 the library GEMM
    with add_rmsnorm, rope_split and silu_mul; 'eager' is the torch glue (fused=False); 'graph' captures one step (after one
    warm-up step, which is the first of the four) and replays it."""
    r = make_runner(B, route != "eager")
    assert torch.equal(r.layers[1]["w_down"][:4].double(), fp64_model["layers"][1]["w_down"][:4])
    for b in range(B):
        r.server.alloc_buffer(STEP_P)
        for li in range(STEP_SHAPE["layers"]):
            k, v = prompt(b, li)
            r.server.fill(li, b, k.to(DEV), v.to(DEV), STEP_P)
    r.pos.copy_(torch.tensor([start_pos(b) for b in range(B)], device=DEV))
    ids = step_ids(B)
    got = []
    for t in range(STEP_STEPS):
        r.ids.copy_(torch.tensor(ids[t], device=DEV)[:, None])
        if route == "graph" and t == 0:
            r.capture(warm=1)                                  # the warm-up step is step 0; the captured step does not run
        elif route == "graph":
            r.replay()
        else:
            r.step()
        torch.cuda.synchronize()
        got.append(r.logits.clone())
    assert r.pos.tolist() == [start_pos(b) + STEP_STEPS for b in range(B)]
    refs = reference_logits(fp64_model, B, ids)
    errs = [rel_err(got[t][b], refs[t][b]) for t in range(STEP_STEPS) for b in range(B)]
    STEP_ERRORS[(route, B)] = max(errs)
    print(f"\n[step numerics] {route} B={B}: largest relative logits error {max(errs):.3e}")
    assert max(errs) < STEP_BAR, errs


@pytest.mark.parametrize("perturb", Fp64Llama.PERTURBATIONS)
def test_step_restatement_is_sensitive(cuda_lib, fp64_model, perturb):
    """Each named mistake in the restatement moves the logits by at least 10x the bar on the inputs of the step test."""
    B = 2
    ids = step_ids(B)
    refs = reference_logits(fp64_model, B, ids)
    bad = reference_logits(fp64_model, B, ids, perturb)
    moved = run_rel_err(bad, refs)
    print(f"\n[step numerics] {perturb}: relative move {moved:.3e}")
    assert moved >= 10 * STEP_BAR, moved
