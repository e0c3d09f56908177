"""The table merge of a window spill (csrc/tables.cu, table_merge_kernel) restated in numpy: offsets and item placement of
CSR(old keys) + new keys must equal a counting-sort rebuild over all keys (csrc/tables.cu, build_segments_kernel).  No GPU: the
kernel itself is checked against a device rebuild in test_gpu_spill.py.
"""
import numpy as np
import pytest


def build(codes, n, K, M, seg_len, S, built=True):
    """build_segments_kernel over keys [0, n): offsets (S, NB+1) absolute in the row, items (M,) uint16 = key - seg_lo.
    built=False: the state of a table that was never built (all offsets zero)."""
    NB = 1 << K
    off = np.zeros((S, NB + 1), dtype=np.int64)
    items = np.full(M, 0xFFFF, dtype=np.int64)   # unwritten slots
    if not built:
        return off, items
    for s in range(S):
        lo, hi = s * seg_len, min(n, s * seg_len + seg_len)
        if lo >= hi:
            off[s] = lo
            continue
        c = codes[lo:hi]
        hist = np.bincount(c, minlength=NB)
        off[s, 1:] = np.cumsum(hist)
        off[s] += lo
        order = np.argsort(c, kind="stable")
        items[lo:lo + (hi - lo)] = order   # key - lo, grouped by bucket
    return off, items


def merge(off, items, codes_new, n_old, K, M, seg_len, S, chunk):
    """table_merge_kernel: one (row, segment) at a time, the old items moved from the top down in chunks of `chunk`
    positions, each chunk read completely before any of it is written."""
    NB = 1 << K
    g = len(codes_new)
    off, items = off.copy(), items.copy()
    for s in range(S):
        seg_lo = s * seg_len
        k0, k1 = max(n_old, seg_lo), min(n_old + g, min(seg_lo + seg_len, M))
        if k0 >= k1:
            if g > 0 and seg_lo >= n_old + g:
                off[s] = seg_lo                               # beyond all keys: every bucket empty, as a build leaves it
            continue
        base0 = off[s, 0]
        ro = off[s] - base0                                   # old offsets relative to the segment
        cn = codes_new[k0 - n_old:k1 - n_old]
        hist = np.bincount(cn, minlength=NB)
        ex = np.concatenate([[0], np.cumsum(hist)])           # exclusive prefix, ex[NB] = total
        it = items[seg_lo:]                                   # view: positions relative to the segment
        top = ro[NB]
        while top > 0:
            lo = max(0, top - chunk)
            p = np.arange(lo, top)
            bucket = np.searchsorted(ro[:NB], p, side="right") - 1   # last bucket whose start is <= p
            sh = ex[bucket]
            vals = it[p].copy()                               # the whole chunk is read ...
            it[p + sh] = vals                                 # ... before any of it is written
            top = lo
        cursor = ex[:NB].copy()
        for j, c in enumerate(cn):
            it[ro[c + 1] + cursor[c]] = k0 + j - seg_lo
            cursor[c] += 1
        # cursor[c] is now the inclusive prefix: new off[c] = seg_lo + ro[c] + ex[c]
        off[s] = seg_lo + ro + ex
    return off, items


def assert_same_tables(off_a, items_a, off_b, items_b, K, S, seg_len):
    NB = 1 << K
    assert np.array_equal(off_a, off_b)
    for s in range(S):
        for c in range(NB):
            a, b = off_a[s, c], off_a[s, c + 1]
            assert sorted(items_a[a:b]) == sorted(items_b[a:b]), (s, c)


CASES = [
    # K, M, seg_len, n_old, g, built
    (10, 1000, 1000, 600, 256, True),          # one segment
    (6, 4096, 1024, 900, 300, True),           # the spill straddles the boundary at 1024
    (6, 4096, 1024, 1024, 200, True),          # new keys start an empty segment (offsets all seg_lo)
    (5, 4096, 1024, 0, 700, False),            # tables never built: n_old = 0, offsets still zero
    (7, 4096, 1024, 0, 1500, False),           # ... and the first spill straddles a boundary
    (15, 70000, 35008, 34000, 2000, True),     # K = 15 across the boundary
    (15, 3000, 3008, 2000, 300, True),         # K = 15, most buckets empty
    (1, 512, 512, 100, 64, True),              # two buckets
    (12, 131072, 65536, 65500, 100, True),     # full-size segments
]


@pytest.mark.parametrize("K,M,seg_len,n_old,g,built", CASES)
@pytest.mark.parametrize("chunk", [2048, 7])
def test_merge_equals_rebuild(K, M, seg_len, n_old, g, built, chunk):
    S = (M + seg_len - 1) // seg_len
    rng = np.random.default_rng(K * 1000 + n_old + g)
    # clustered codes: some buckets hold many keys, many hold none
    codes = np.minimum(rng.geometric(0.02, size=n_old + g) - 1, (1 << K) - 1) ^ rng.integers(0, 2, n_old + g)
    codes = np.clip(codes, 0, (1 << K) - 1)
    off0, items0 = build(codes, n_old, K, M, seg_len, S, built=built)
    off1, items1 = merge(off0, items0, codes[n_old:], n_old, K, M, seg_len, S, chunk)
    off_r, items_r = build(codes, n_old + g, K, M, seg_len, S)
    assert_same_tables(off1, items1, off_r, items_r, K, S, seg_len)


def test_two_merges_in_a_row():
    K, M, seg_len = 8, 2048, 1024
    S = 2
    rng = np.random.default_rng(3)
    codes = rng.integers(0, 1 << K, size=1400)
    off, items = build(codes, 800, K, M, seg_len, S)
    off, items = merge(off, items, codes[800:1100], 800, K, M, seg_len, S, 64)
    off, items = merge(off, items, codes[1100:1400], 1100, K, M, seg_len, S, 64)
    off_r, items_r = build(codes, 1400, K, M, seg_len, S)
    assert_same_tables(off, items, off_r, items_r, K, S, seg_len)


def test_shift_never_decreases_with_position():
    """The in-place move is safe because old position p goes to p + ex[bucket(p)] with ex non-decreasing: destinations are
    strictly increasing and never below their source."""
    rng = np.random.default_rng(4)
    for K in (1, 4, 10, 15):
        NB = 1 << K
        hist_old = rng.integers(0, 3, NB)
        ro = np.concatenate([[0], np.cumsum(hist_old)])
        ex = np.concatenate([[0], np.cumsum(rng.integers(0, 2, NB))])
        p = np.arange(ro[NB])
        dst = p + ex[np.searchsorted(ro[:NB], p, side="right") - 1]
        assert np.all(np.diff(dst) > 0) and np.all(dst >= p)

