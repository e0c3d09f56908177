"""A host restatement of the filtered sampling rule of mpig_aux_sample_filtered and mpig_aux_verify_sample_filtered
(mpig_sample_filters in include/magicpig_b200_aux.h): the penalties in numpy float32 in the stated operation order, the prefix
truncation (top-k, top-p over the top-k set, min-p) in Python integers, and the draw and acceptance through sample_rule's and
spec_rule's helpers.

`mistake` names a wrong rule the tests show the contract rejects:
  "p_from_S"          the top-p threshold taken from the full mass S instead of S_k
  "minp_first"        min-p applied before the top-p renormalisation (vLLM's order): thr = floor(p * mass of the top-k and min-p set)
  "minp_sum"          min-p relative to the sum: W_i >= floor(min_p * S) instead of floor(min_p * 2^40)
  "pos_times_r"       positive logits multiplied by r instead of divided
  "freq_after_temp"   the frequency penalty subtracted after the temperature (l1 / T - f c, i.e. f c scaled by T)
  "prompt_counted"    the presence and frequency penalties count a prompt token as one occurrence
  "ignore_drafts"     verification row t does not count the drafts d_1 .. d_t
  "topk_ties_high"    the top-k order breaks ties by the higher index first
"""
from __future__ import annotations

import numpy as np

from . import sample_rule as sr
from . import spec_rule as spr

COUNT_MASK = 0x7FFFFFFF
PROMPT_BIT = 1 << 31
NEUTRAL = dict(top_k=0, min_p=0.0, repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0)


def device_values(top_k=0, min_p=0.0, repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0):
    """The values as the device reads them: fp32, a non-finite or <= 0 r taken as 1, a non-finite pr or f as 0."""
    f32 = lambda v: np.float32(v)  # noqa: E731
    r, pr, f = f32(repetition_penalty), f32(presence_penalty), f32(frequency_penalty)
    r = r if np.isfinite(r) and r > 0 else np.float32(1)
    pr = pr if np.isfinite(pr) else np.float32(0)
    f = f if np.isfinite(f) else np.float32(0)
    return dict(top_k=int(np.int32(top_k)), min_p=f32(min_p), r=r, pr=pr, f=f, pen=not (r == 1 and f == 0 and pr == 0))


def draft_counts(drafts, V: int) -> np.ndarray:
    """The occurrences of each token among the drafts d_1 .. d_t (ids outside [0, V) are no token)."""
    c = np.zeros(V, dtype=np.int64)
    for d in drafts:
        if 0 <= int(d) < V:
            c[int(d)] += 1
    return c


def penalised(logits, table_row, extra, vals, T: float = 1.0, mistake=None) -> np.ndarray:
    """l3 of every token: table_row the (V,) uint32 entries, extra the drafts' counts (None: none).  numpy float32 rounds each
    operation to nearest as the kernel's __fdiv_rn / __fmul_rn / __fsub_rn do."""
    l = np.asarray(logits, dtype=np.float32)
    if not vals["pen"]:
        return l.copy()
    e = np.asarray(table_row, dtype=np.uint64)[: l.shape[0]]
    c = (e & COUNT_MASK).astype(np.int64) + (0 if extra is None else np.asarray(extra, dtype=np.int64))
    prompt = (e >> 31).astype(bool)
    seen = prompt | (c > 0)
    cp = c + prompt if mistake == "prompt_counted" else c
    r, f, pr = vals["r"], vals["f"], vals["pr"]
    with np.errstate(over="ignore", invalid="ignore"):
        pos = l * r if mistake == "pos_times_r" else l / r
        l1 = np.where(seen, np.where(l > 0, pos, l * r), l).astype(np.float32)
        fc = f * cp.astype(np.float32)
        if mistake == "freq_after_temp":
            fc = (fc * np.float32(T)).astype(np.float32)
        l2 = (l1 - fc).astype(np.float32)
        l3 = np.where(cp > 0, l2 - pr, l2).astype(np.float32)
    return l3


def truncate(W, top_p: float, vals, mistake=None):
    """The kept set of a sampled row on fixed-point weights W: the first K = max(1, min(n_k, n_p, n_m)) tokens of the order.
    Returns (keep mask, dict(S, S_k, thr, n_k, n_p, n_m, K))."""
    W = np.asarray(W, dtype=np.int64)
    V = W.shape[0]
    order = sr.sorted_order(W, "ties_high" if mistake == "topk_ties_high" else None)
    Wo = W[order]
    incl = np.cumsum(Wo)   # exact: S < V 2^41 < 2^63
    before = incl - Wo
    S = int(incl[-1])
    n_k = min(vals["top_k"], V) if vals["top_k"] > 0 else V
    S_k = int(incl[n_k - 1])
    Wm = sr.nucleus_threshold(vals["min_p"], S if mistake == "minp_sum" else 1 << sr.FRAC_BITS)
    n_m = int((Wo >= Wm).sum())
    base = S if mistake == "p_from_S" else S_k
    if mistake == "minp_first":
        base = int(incl[min(n_k, n_m) - 1]) if min(n_k, n_m) else 0
    p32 = float(np.float32(top_p))
    thr = sr.nucleus_threshold(p32, base)
    n_p = int((before <= thr).sum()) if p32 < 1 else V   # the kernel selects only for p < 1 (as the unfiltered rule)
    K = max(1, min(n_k, n_p, n_m))
    keep = np.zeros(V, dtype=bool)
    keep[order[:K]] = True
    return keep, dict(S=S, S_k=S_k, thr=thr, n_k=n_k, n_p=n_p, n_m=n_m, K=K)


def row_kind(logits, l3, T):
    """sample_rule.row_kind on the raw and the penalised logits: invalid if either holds a NaN or +inf (or no finite value)."""
    if sr.row_kind(logits, T) == sr.INVALID or sr.row_kind(l3, T) == sr.INVALID:
        return sr.INVALID
    return sr.row_kind(l3, T)


def sample_row(logits, T, p, vals, table_row, seed, offset, row, W=None, mistake=None):
    """One row of mpig_aux_sample_filtered: (token, debug 8-tuple).  W: the fixed-point weights to use (default: fp64 of l3)."""
    l3 = penalised(logits, table_row, None, vals, T, mistake)
    kind = row_kind(logits, l3, T)
    if kind == sr.INVALID:
        return 0, (0,) * 8
    if kind == sr.GREEDY:
        return int(np.argmax(l3)), (0, 0, 0, 1, 0, 0, 0, 0)
    if W is None:
        W = sr.fixed_point(sr.weights_fp64(l3, T))
    W = np.asarray(W, dtype=np.int64)
    keep, info = truncate(W, p, vals, mistake)
    kept_w = np.where(keep, W, 0)
    S_keep = int(kept_w.sum())
    target = (sr.draw_word(seed, offset, row) * S_keep) >> 64
    token = int(np.searchsorted(np.cumsum(kept_w), target, side="right"))
    return token, (info["S"], info["thr"], S_keep, info["K"], int(target), info["n_k"], info["S_k"], info["n_m"])


def verify_row(logits, T, p, vals, table_row, drafts_before, seed, offset, b, t, d, W=None, mistake=None):
    """Row (b, t) of mpig_aux_verify_sample_filtered: (accept, final, invalid, debug 12-tuple).  drafts_before: d_1 .. d_t."""
    V = len(logits)
    extra = None if mistake == "ignore_drafts" else draft_counts(drafts_before, V)
    l3 = penalised(logits, table_row, extra, vals, T, mistake)
    kind = row_kind(logits, l3, T)
    if kind == sr.INVALID:
        return False, 0, True, (0,) * 12
    am = int(np.argmax(l3))
    if kind == sr.GREEDY:
        acc = d is not None and int(d) == am
        return acc, am, False, (0, 0, 0, 1, 0, 0, int(acc), 0, 0, 0, 0, 0)
    if W is None:
        W = sr.fixed_point(sr.weights_fp64(l3, T))
    W = np.asarray(W, dtype=np.int64)
    keep, info = truncate(W, p, vals, mistake)
    r0, r_acc = spr.philox_word(seed, offset, b, 0), spr.philox_word(seed, offset, b, t + 1)
    accept, final, (S_keep, W_d, kept_d, acc_target, S_res) = row_from_keep(W, keep, r0, r_acc, d, am)
    dbg = (info["S"], info["thr"], S_keep, info["K"], (r0 * S_keep) >> 64, W_d, int(kept_d), acc_target, S_res, info["n_k"],
           info["S_k"], info["n_m"])
    return accept, final, False, dbg


def row_from_keep(W, keep, r0: int, r_acc: int, d, argmax: int):
    """The acceptance and the residual draw of a sampled row on its kept set, as spec_rule.row_from_weights does them on the
    nucleus: (accept, final, (S_keep, W_d, kept_d, acc_target, S_res)).  r0 / r_acc: the residual and acceptance words."""
    W = np.asarray(W, dtype=np.int64)
    kept_w = np.where(keep, W, 0)
    S_keep = int(kept_w.sum())
    has_d = d is not None and 0 <= int(d) < W.shape[0]
    W_d = int(W[d]) if has_d else 0
    kept_d = bool(keep[d]) if has_d else False
    acc_target = (r_acc * S_keep) >> 64 if has_d else 0
    accept = kept_d and acc_target < W_d
    res = kept_w.copy()
    if kept_d:
        res[d] = 0
    S_res = int(res.sum())
    final = argmax if S_res == 0 else int(np.searchsorted(np.cumsum(res), (r0 * S_res) >> 64, side="right"))
    return accept, final, (S_keep, W_d, kept_d, acc_target, S_res)


def request(logits, T_temp, p, vals, table_row, seed, offset, b, ids_row, W_rows=None, mistake=None, **book):
    """One request of a filtered verification step: spec_rule.resolve() over verify_row()'s rows, plus the table after the step
    ('table': the counts incremented for each appended token).  Returns resolve()'s dict plus 'rows' and 'table'."""
    Tn, V = len(logits), len(logits[0])
    drafts = [int(x) for x in ids_row[1:Tn]]
    rows = []
    for t in range(Tn):
        d = drafts[t] if t < Tn - 1 else None
        d = d if d is not None and 0 <= d < V else None
        rows.append(verify_row(logits[t], T_temp, p, vals, table_row, drafts[:t], seed, offset, b, t, d,
                               None if W_rows is None else W_rows[t], mistake))
    out = spr.resolve([r[:3] for r in rows], drafts, **book)
    out["rows"] = rows
    tab = np.asarray(table_row, dtype=np.uint64).copy()
    for tok in out["emitted"]:
        tab[tok] += 1
    out["table"] = tab
    return out
