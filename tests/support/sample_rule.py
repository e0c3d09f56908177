"""A host restatement of the sampling contract of mpig_aux_sample (include/magicpig_b200_aux.h, csrc/aux_sample.cu): Philox4x32-10
and the integer stages that follow the weights, in Python integers.  The weights come either from fp64 (`weights_fp64`) or from
the kernel itself (its debug_w output, `fixed_point`), so the same stages check the kernel bitwise and against fp64.

`mistake` names a wrong rule the tests show the contract rejects:
  "sorted_draw"     draw in the nucleus's sorted order instead of index order
  "inclusive"       keep a token when the mass up to and including it is <= floor(p S)
  "ties_high"       break ties by the higher index first
  "target32"        a 32-bit target: umulhi32 of r's low word and S_keep, scaled by 2^-32
"""
from __future__ import annotations

import math

import numpy as np

MASK32 = 0xFFFFFFFF
PHILOX_M = (0xD2511F53, 0xCD9E8D57)
PHILOX_W = (0x9E3779B9, 0xBB67AE85)
LOG2E_F32 = float(np.float32(1.44269504))
FRAC_BITS = 40
GREEDY, INVALID = "greedy", "invalid"


def philox4x32_10(ctr, key):
    """curand_Philox4x32_10(counter (c0, c1, c2, c3), key (k0, k1)) -> four 32-bit words."""
    c0, c1, c2, c3 = (int(x) & MASK32 for x in ctr)
    k0, k1 = (int(x) & MASK32 for x in key)
    for _ in range(10):
        p0, p1 = PHILOX_M[0] * c0, PHILOX_M[1] * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & MASK32, (p0 >> 32) ^ c3 ^ k1, p0 & MASK32
        k0, k1 = (k0 + PHILOX_W[0]) & MASK32, (k1 + PHILOX_W[1]) & MASK32
    return c0, c1, c2, c3


def draw_word(seed: int, offset: int, row: int) -> int:
    """r: the first two Philox words of counter (offset lo, offset hi, row, 0) under key (seed lo, seed hi), as x | y << 32."""
    x, y, _, _ = philox4x32_10((offset & MASK32, (offset >> 32) & MASK32, row, 0), (seed & MASK32, (seed >> 32) & MASK32))
    return x | (y << 32)


def row_kind(logits: np.ndarray, T: float) -> str | None:
    """INVALID for a row with a NaN or +inf logit or none finite, GREEDY for T <= 0 or NaN, None for a sampled row."""
    l = np.asarray(logits, dtype=np.float32)
    if np.isnan(l).any() or np.isposinf(l).any() or not np.isfinite(l).any():
        return INVALID
    if not float(T) > 0:
        return GREEDY
    return None


def weights_fp64(logits: np.ndarray, T: float) -> np.ndarray:
    """w_i = exp((l_i - m) / T) in fp64 from the fp32 logits and the fp32 temperature; -inf logits weigh 0."""
    l = np.asarray(logits, dtype=np.float32).astype(np.float64)
    m = l.max()
    with np.errstate(invalid="ignore", over="ignore"):
        w = np.exp((l - m) / float(np.float32(T)))
    w[np.isneginf(l)] = 0.0
    return w


def fixed_point(w: np.ndarray) -> np.ndarray:
    """W_i = floor(w_i * 2^40) as int64 (exact for fp32 or fp64 w in [0, 1])."""
    return np.floor(np.asarray(w, dtype=np.float64) * 2.0 ** FRAC_BITS).astype(np.int64)


def nucleus_threshold(p: float, S: int) -> int:
    """floor(p * S) from p's 24-bit significand: p >= 1 -> S, p <= 0 (or NaN) -> 0."""
    p = float(np.float32(p))
    if p >= 1:
        return S
    if not p > 0:
        return 0
    mant, e = math.frexp(p)
    m24 = int(mant * (1 << 24))
    return (m24 * S) >> (24 - e)


def sorted_order(W: np.ndarray, mistake: str | None = None) -> np.ndarray:
    """The nucleus order: W descending, the lower index first on ties ("ties_high": the higher first)."""
    idx = np.arange(W.shape[0])
    return np.lexsort((-idx if mistake == "ties_high" else idx, -W))


def keep_mask(W: np.ndarray, thr: int, mistake: str | None = None) -> np.ndarray:
    """Token i is kept iff the W of the tokens ordered before it sum to <= thr."""
    order = sorted_order(W, mistake)
    incl = np.cumsum(W[order])
    before = incl - W[order]
    keep = np.zeros(W.shape[0], dtype=bool)
    keep[order] = (incl if mistake == "inclusive" else before) <= thr
    if mistake == "inclusive" and not keep.any():
        keep[order[0]] = True
    return keep


def sample_from_weights(W: np.ndarray, p: float, r: int, mistake: str | None = None):
    """The integer stages of one sampled row: (token, (S, floor(p S), S_keep, kept count, target), keep mask)."""
    W = np.asarray(W, dtype=np.int64)
    S = int(W.sum())
    thr = nucleus_threshold(p, S)
    keep = keep_mask(W, thr, mistake)
    kept_w = np.where(keep, W, 0)
    S_keep = int(kept_w.sum())
    if mistake == "target32":
        target = (((r & MASK32) * S_keep) >> 32)
    else:
        target = (r * S_keep) >> 64
    if mistake == "sorted_draw":
        order = sorted_order(W)
        cum = np.cumsum(kept_w[order])
        token = int(order[int(np.searchsorted(cum, target, side="right"))])
    else:
        cum = np.cumsum(kept_w)
        token = int(np.searchsorted(cum, target, side="right"))
    return token, (S, thr, S_keep, int(keep.sum()), int(target)), keep


def sample_row(logits, T, p, seed, offset, row, W=None, mistake=None):
    """The contract for one row: (token, debug tuple).  W: the fixed-point weights to use (default: from fp64 weights)."""
    kind = row_kind(logits, T)
    if kind == INVALID:
        return 0, (0, 0, 0, 0, 0)
    if kind == GREEDY:
        return int(np.argmax(np.asarray(logits, dtype=np.float32))), (0, 0, 0, 1, 0)
    if W is None:
        W = fixed_point(weights_fp64(logits, T))
    token, dbg, _ = sample_from_weights(W, p, draw_word(seed, offset, row), mistake)
    return token, dbg


def weight_rel_bound(logits: np.ndarray, T: float) -> np.ndarray:
    """Relative error bound of the kernel's fp32 w_i = exp2f((l_i - m) * (1.44269504f / T)) against fp64 exp((l_i - m) / T).
    The argument x = (l_i - m) log2(e) / T is off by at most 4 roundings of 2^-24 each (l_i - m, the fp32 log2 e, the division and
    the product), |dx| <= |x| 2^-22; exp2f adds at most 2 ulp (2^-22 relative).  So |dw| / w <= 2^-22 (1 + |x| ln 2) to first
    order; the bound doubles it for the second-order terms."""
    l = np.asarray(logits, dtype=np.float32).astype(np.float64)
    with np.errstate(invalid="ignore"):
        x = np.abs((l - l.max()) / float(np.float32(T))) * math.log2(math.e)
    x[~np.isfinite(x)] = 0.0
    return 2.0 ** -21 * (1.0 + x * math.log(2.0))


def allowed_tokens(logits, T, p, r, W64, rel):
    """The tokens a draw may take when the kernel's weights are within `rel` of the fp64 weights W64 / 2^40: delta_i = W64_i rel + 1
    per token (the relative error and the floor), E = sum delta_i bounds |dS|, |d floor(p S)| and every prefix's shift.  A token's
    keep status is ambiguous where its prefix lies within 2E of the threshold; A = 2E + the mass of those tokens bounds |dS_keep|
    and every kept prefix's shift, so the target's interval in index order widens by 2A.  Returns the set of admissible ids."""
    W64 = np.asarray(W64, dtype=np.int64)
    delta = np.where(np.asarray(logits, dtype=np.float32) > -np.inf, W64 * rel + 1.0, 0.0)
    E = float(delta.sum())
    S = int(W64.sum())
    thr = nucleus_threshold(p, S)
    order = sorted_order(W64)
    before = np.empty_like(W64)
    before[order] = np.cumsum(W64[order]) - W64[order]
    keep = before <= thr
    ambiguous = np.abs(before.astype(np.float64) - thr) <= 2 * E
    A = 2 * E + float(W64[ambiguous].sum())
    kept_w = np.where(keep, W64, 0)
    cum = np.cumsum(kept_w).astype(np.float64)
    target = float((r * int(kept_w.sum())) >> 64)
    lo, hi = cum - kept_w, cum
    ok = (keep | ambiguous) & (W64 + delta > 0) & (lo - 2 * A <= target) & (target < hi + 2 * A)
    return set(np.nonzero(ok)[0].tolist())
