"""A host restatement of the speculative-decoding contracts of include/magicpig_b200_aux.h: mpig_aux_verify_sample (acceptance of a
verification step's drafts, the residual draw, drop and the history bookkeeping) and mpig_aux_ngram_draft (prompt-lookup drafts).
The row stages are sample_rule's; this module adds what the verification rule puts on top of them.

`mistake` names a wrong rule the tests show the contract rejects:
  "no_exclude"   the residual draw does not exclude the rejected draft (draws from the whole kept set)
  "reuse_word"   the residual draw reuses the acceptance word r_acc instead of the word at counter (.., b, 0)
  "le"           accept when umulhi64(r_acc, S_keep) <= W_d instead of <
  "drop_off"     drop = T - k instead of T - 1 - k
  "next_row"     the final token taken from row k + 1 instead of row k
"""
from __future__ import annotations

import numpy as np

from . import sample_rule as sr

MASK32 = sr.MASK32


def philox_word(seed: int, offset: int, row: int, word: int) -> int:
    """The first two Philox words of counter (offset lo, offset hi, row, word) under key (seed lo, seed hi), as x | y << 32."""
    x, y, _, _ = sr.philox4x32_10((offset & MASK32, (offset >> 32) & MASK32, row, word), (seed & MASK32, (seed >> 32) & MASK32))
    return x | (y << 32)


def row_from_weights(W, p: float, r0: int, r_acc: int, d, mistake=None, argmax: int | None = None):
    """One sampled row on fixed-point weights W: (accept, final token if acceptance ends here, debug 9-tuple).  d: the draft this row
    checks (None: none, or an id outside [0, V)); r0 / r_acc: the residual and acceptance words."""
    W = np.asarray(W, dtype=np.int64)
    V = W.shape[0]
    S = int(W.sum())
    thr = sr.nucleus_threshold(p, S)
    keep = sr.keep_mask(W, thr)
    kept_w = np.where(keep, W, 0)
    S_keep = int(kept_w.sum())
    has_d = d is not None and 0 <= int(d) < V
    W_d = int(W[d]) if has_d else 0
    kept_d = bool(keep[d]) if has_d else False
    acc_target = (r_acc * S_keep) >> 64 if has_d else 0
    accept = kept_d and (acc_target <= W_d if mistake == "le" else acc_target < W_d)
    res = kept_w.copy()
    if kept_d and mistake != "no_exclude":
        res[d] = 0
    S_res = int(res.sum())
    target = ((r_acc if mistake == "reuse_word" else r0) * S_res) >> 64
    if S_res == 0:
        final = int(argmax if argmax is not None else int(np.argmax(W)))
    else:   # the index-order scan: the first index at which the running residual sum exceeds target (sums < 2^63)
        final = int(np.searchsorted(np.cumsum(res), target, side="right"))
    dbg = (S, thr, S_keep, int(keep.sum()), (r0 * S_keep) >> 64, W_d, int(kept_d), acc_target, S_res)
    return accept, final, dbg


def row(logits, T, p, seed, offset, b, t, d, W=None, mistake=None):
    """Row (b, t) of a verification step: (accept, final, invalid, debug 9-tuple).  W: the fixed-point weights (default: fp64)."""
    kind = sr.row_kind(logits, T)
    if kind == sr.INVALID:
        return False, 0, True, (0,) * 9
    am = int(np.argmax(np.asarray(logits, dtype=np.float32)))
    if kind == sr.GREEDY:
        acc = d is not None and int(d) == am
        return acc, am, False, (0, 0, 0, 1, 0, 0, int(acc), 0, 0)
    if W is None:
        W = sr.fixed_point(sr.weights_fp64(logits, T))
    r0 = philox_word(seed, offset, b, 0)
    r_acc = philox_word(seed, offset, b, t + 1)
    acc, final, dbg = row_from_weights(W, p, r0, r_acc, d, mistake, argmax=am)
    return acc, final, False, dbg


def resolve(rows, drafts, done=False, length=0, limit=1 << 30, eos=(), mistake=None):
    """The per-request step after its rows: rows = [(accept, final, invalid), ...] (T of them), drafts = [d_1 .. d_{T-1}].
    drop = T - 1 - k, except T - (tokens appended) for a request that ends in this step and T for one already done.
    Returns dict(k, final, drop, emitted (appended tokens), done, length, invalid, counted)."""
    T, was_done = len(rows), done
    k = 0
    while k < T - 1 and rows[k][0]:
        k += 1
    src = min(k + 1, T - 1) if mistake == "next_row" else k
    final, invalid = rows[src][1], rows[src][2]
    emitted = []
    if not done:
        for tok in list(drafts[:k]) + [final]:
            if done:
                break
            if length < limit:
                emitted.append(int(tok))
                length += 1
            if int(tok) in eos or length >= limit:
                done = True
    # the rows that stay: none for a request already done, the emitted tokens' for one that ends here, k + 1 otherwise
    keep = 0 if was_done else (len(emitted) if done else k + 1)
    drop = T - keep + (1 if mistake == "drop_off" else 0)
    return dict(k=k, final=final, drop=drop, emitted=emitted, done=done, length=length, invalid=invalid, counted=not was_done)


def request(logits, T_temp, p, seed, offset, b, ids_row, W_rows=None, mistake=None, **book):
    """One request of a verification step: logits (T, V), ids_row[0 .. T) the step's inputs.  W_rows: per-row fixed-point weights
    (None: fp64).  book: done / length / limit / eos for resolve().  Returns resolve()'s dict plus 'rows' (each row's 4-tuple)."""
    T = len(logits)
    V = len(logits[0])
    rows = []
    for t in range(T):
        d = int(ids_row[t + 1]) if t < T - 1 else None
        d = d if d is not None and 0 <= d < V else None
        rows.append(row(logits[t], T_temp, p, seed, offset, b, t, d, None if W_rows is None else W_rows[t], mistake))
    out = resolve([r[:3] for r in rows], [int(x) for x in ids_row[1:T]], mistake=mistake, **book)
    out["rows"] = rows
    return out


# ---- prompt lookup -----------------------------------------------------------------------------------------------------------
def ngram_match_lengths(h, g_max: int) -> np.ndarray:
    """m(e) for e in [0, n - 2]: the largest m <= g_max with h[e - i] == h[n - 1 - i] for all i < m."""
    h = np.asarray(h, dtype=np.int64)
    n = h.shape[0]
    if n < 2:
        return np.zeros(0, dtype=np.int64)
    e = np.arange(n - 1)
    m = np.zeros(n - 1, dtype=np.int64)
    alive = np.ones(n - 1, dtype=bool)
    for i in range(g_max):
        ok = alive & (e - i >= 0)
        ok[ok] = h[e[ok] - i] == h[n - 1 - i]
        alive = ok
        m += alive
    return m


def ngram_choice(h, g_min: int = 1, g_max: int = 3):
    """e*: the end maximising (m(e), e) among m(e) >= g_min, or None."""
    m = ngram_match_lengths(h, g_max)
    ok = np.nonzero(m >= g_min)[0]
    if ok.size == 0:
        return None
    best = m[ok].max()
    return int(ok[m[ok] == best].max())


def ngram_drafts(h, T: int, g_min: int = 1, g_max: int = 3) -> list:
    """The T - 1 drafts: h'[e* + 1 + i] with h' = h followed by the drafts; h[n - 1] each when nothing matches (0 when n = 0)."""
    h = [int(x) for x in h]
    n = len(h)
    e = ngram_choice(h, g_min, g_max)
    if e is None:
        return [h[-1] if n else 0] * (T - 1)
    ext = list(h)
    for i in range(T - 1):
        ext.append(ext[e + 1 + i])
    return ext[n:]
