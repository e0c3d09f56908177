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

import numpy as np
import pytest
import torch

from tests.support.fp64 import bf16_rne
from tests.support.step_rule import (OFF_MARGIN, Fp64Llama, assert_rule, gemv_ref, neighbours, prompt_kv, rel_err, rmsnorm_ref,
                                     rope_cands, run_reference, run_rel_err, ss_roundings_add_rmsnorm, ss_roundings_prologue,
                                     swiglu_cands)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MPIG_EINVAL, MPIG_EUNSUPPORTED = -1, -5


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


def prompt(b: int, layer: int):
    return prompt_kv(torch.Generator().manual_seed(1000 + 10 * b + layer), STEP_P, STEP_SHAPE["Hkv"])


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
