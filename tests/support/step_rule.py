"""The interval rule of tests/test_gpu_step_numerics.py and its fp64 restatements of the decode step's kernels and of a whole
Llama step (also checked without a GPU by tests/test_step_numerics_cpu.py)."""
import math

import numpy as np
import torch

from tests.support.fp64 import bf16_rne

U = 2.0 ** -24                 # fp32 unit roundoff
TINY = 2.0 ** -149             # fp32 subnormal step: absolute floor of every bound
OFF_MARGIN = {}                # kernel -> largest number of elements seen per call that differ from bf16(ref) inside the rule


# ------------------------------------------------------------------------------------------------
# bf16 rounding and the interval rule (device-agnostic torch, fp64)
# ------------------------------------------------------------------------------------------------
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
# the step against an fp64 Llama
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


def prompt_kv(g: torch.Generator, P: int, Hkv: int):
    """(k, v) (P, Hkv, 128) bf16 of a prompt on which the step's attention matters: a short prompt, so the token being
    decoded carries a large share of the attention, and keys three times larger on the 8 highest-frequency RoPE pairs (dims
    0..7 and 64..71), so that the scores depend on the rotation of q."""
    scale = torch.ones(128)
    scale[0:8] = scale[64:72] = 3.0
    k = (torch.randn((P, Hkv, 128), generator=g) * scale).bfloat16()
    v = torch.randn((P, Hkv, 128), generator=g).bfloat16()
    return k, v


def run_rel_err(got, ref) -> float:
    """Relative distance between the logits of two runs (every step and request)."""
    return rel_err(torch.stack(list(got)), torch.stack(list(ref)))


def run_reference(m, prompts, start, ids, perturb=None):
    """Logits of every step: prompts[b][layer] = (k, v) (P, Hkv, d), start[b] = the prompt's last position, ids[t][b]."""
    B = len(prompts)
    ref = Fp64Llama(m, B, perturb)
    for b in range(B):
        for li, (k, v) in enumerate(prompts[b]):
            ref.prefill(b, li, k, v)
    return [ref.step(ids[t], [start[b] + 1 + t for b in range(B)]) for t in range(len(ids))]
