"""Compaction of a shared context restated in numpy on the segmented CSR tables (uint16 items, seg_len key segments): the live
list, table_truncate_kernel's stable in-place partition and table_merge_kernel's in-place merge, checked against a rebuild over
the compacted keys.  Covered: private keys on both sides of a segment boundary, live keys moving into a lower segment, a slot whose
keys are all live, one whose keys are all dead, and buckets whose private items are not a suffix."""
import numpy as np
import pytest

NB = 64


def geometry(M):
    S = -(-M // 65536)
    return S, ((-(-M // S)) + 63) & ~63


def build(codes, M):
    """build_segments_kernel: per segment, a counting sort of its keys by code"""
    S, seg_len = geometry(M)
    off = np.zeros((S, NB + 1), np.int64)
    items = np.zeros(M, np.uint16)
    n = len(codes)
    for s in range(S):
        lo, hi = s * seg_len, min(n, s * seg_len + seg_len)
        if lo >= hi:
            off[s] = lo
            continue
        keys = np.arange(lo, hi)
        order = np.argsort(codes[lo:hi], kind="stable")
        hist = np.bincount(codes[lo:hi], minlength=NB)
        off[s, 1:] = np.cumsum(hist)
        off[s] += lo
        items[lo:lo + len(keys)] = (keys[order] - lo).astype(np.uint16)
    return off, items


def live_list(vis, n_priv):
    """compact_live_kernel: the ascending offsets whose visibility word is not 0"""
    return np.flatnonzero(vis[:n_priv] != 0)


def truncate(off, items, lo, hi, M):
    """table_truncate_kernel: drop the items of keys >= lo from the segments holding keys of [lo, hi), a stable partition
    in place (kept items move down in ascending chunks, each read before it is written)"""
    S, seg_len = geometry(M)
    for s in range(S):
        seg_lo = s * seg_len
        if max(lo, seg_lo) >= min(hi, seg_lo + seg_len, M):
            continue
        o = off[s] - off[s, 0]
        it = items[seg_lo:]
        cnt, lim = o[NB], lo - seg_lo
        kc = np.zeros(NB + 1, np.int64)
        for p in range(cnt):
            if it[p] < lim:
                kc[np.searchsorted(o, p, side="right") - 1] += 1
        new = np.concatenate([[0], np.cumsum(kc[:NB])])
        out, chunk = 0, 37   # any chunk size: a kept item never lands above its source
        for p0 in range(0, cnt, chunk):
            v = it[p0:min(cnt, p0 + chunk)].copy()
            keep = v[v < lim]
            it[out:out + len(keep)] = keep
            out += len(keep)
        off[s] = seg_lo + new


def merge(off, items, codes_new, n_old, M):
    """table_merge_kernel: old items shifted top chunk first by the exclusive prefix of the new codes of the buckets before
    theirs, new keys behind the old items of their bucket"""
    S, seg_len = geometry(M)
    g = len(codes_new)
    for s in range(S):
        seg_lo = s * seg_len
        seg_hi = min(seg_lo + seg_len, M)
        k0, k1 = max(n_old, seg_lo), min(n_old + g, seg_hi)
        if k0 >= k1:
            if g > 0 and seg_lo >= n_old + g:
                off[s] = seg_lo
            continue
        it = items[seg_lo:]
        oo = off[s] - off[s, 0]
        cn = codes_new[k0 - n_old:k1 - n_old]
        ex = np.concatenate([[0], np.cumsum(np.bincount(cn, minlength=NB))])
        for p in range(oo[NB] - 1, -1, -1):
            it[p + ex[np.searchsorted(oo, p, side="right") - 1]] = it[p]
        cur = ex[:NB].copy()
        for k, c in zip(range(k0, k1), cn):
            it[oo[c + 1] + cur[c]] = k - seg_lo
            cur[c] += 1
        off[s] = seg_lo + oo + ex


def buckets(off, items, M):
    S, seg_len = geometry(M)
    return [[sorted(s * seg_len + items[off[s, c]:off[s, c + 1]].astype(np.int64)) for c in range(NB)] for s in range(S)]


def compact(codes, n_prompt, vis, M, shuffle=None):
    """Spill-built tables of n_prompt prompt keys and len(vis) private keys (merged in three spills), then the compaction.
    Returns the compacted tables, the kept key order and the count reclaimed."""
    n = len(codes)
    off, items = build(codes[:n_prompt], M)
    cuts = [n_prompt, n_prompt + (n - n_prompt) // 3, n_prompt + 2 * (n - n_prompt) // 3, n]
    for a, b in zip(cuts, cuts[1:]):
        merge(off, items, codes[a:b], a, M)
    assert buckets(off, items, M) == buckets(*build(codes, M), M)   # the spill side agrees with a build
    if shuffle is not None:   # any order inside a bucket: the truncate relies on none
        S, _ = geometry(M)
        for s in range(S):
            for c in range(NB):
                seg = items[off[s, c]:off[s, c + 1]]
                shuffle.shuffle(seg)
    live = live_list(vis, n - n_prompt)
    truncate(off, items, n_prompt, n, M)
    merge(off, items, codes[n_prompt + live], n_prompt, M)
    order = np.concatenate([np.arange(n_prompt), n_prompt + live])
    return off, items, order, (n - n_prompt) - len(live)


def check(codes, n_prompt, vis, M, shuffle=None):
    off, items, order, dead = compact(codes, n_prompt, vis, M, shuffle)
    ref_off, ref_items = build(codes[order], M)
    assert buckets(off, items, M) == buckets(ref_off, ref_items, M)
    assert np.array_equal(off, ref_off), "offsets differ from a build over the compacted keys"
    return dead


@pytest.mark.parametrize("seed", [0, 1])
def test_live_keys_cross_a_segment_boundary(seed):
    """M = 70 000: two segments of 35 008 keys.  The prompt ends 6 keys below the boundary; the first 40 private keys are dead,
    so the live ones in the upper segment move down into the lower one."""
    rng = np.random.default_rng(seed)
    M = 70000
    S, seg_len = geometry(M)
    assert S == 2
    n_prompt, n_priv = seg_len - 6, 300
    codes = rng.integers(0, NB, n_prompt + n_priv)
    vis = rng.integers(0, 2, n_priv).astype(np.uint32) << rng.integers(0, 8, n_priv).astype(np.uint32)
    vis[:40] = 0
    assert check(codes, n_prompt, vis, M) == int((vis == 0).sum())


def test_private_items_not_a_suffix():
    rng = np.random.default_rng(5)
    M = 70000
    _, seg_len = geometry(M)
    n_prompt, n_priv = seg_len - 100, 400
    codes = rng.integers(0, NB, n_prompt + n_priv)
    vis = (rng.random(n_priv) < 0.4).astype(np.uint32)
    assert check(codes, n_prompt, vis, M, shuffle=rng) == int((vis == 0).sum())


def test_every_key_live():
    rng = np.random.default_rng(7)
    M = 4096
    codes = rng.integers(0, NB, 3000)
    vis = np.full(500, 3, np.uint32)
    assert check(codes, 2500, vis, M) == 0


def test_no_key_live():
    """Every private key dead: the tables become the prompt's build, including the offsets seg_lo past the keys."""
    rng = np.random.default_rng(9)
    M = 70000
    _, seg_len = geometry(M)
    codes = rng.integers(0, NB, seg_len + 900)
    vis = np.zeros(1000, np.uint32)
    assert check(codes, seg_len - 100, vis, M) == 1000


def test_live_list():
    vis = np.array([0, 4, 0, 0, 1, 6, 0, 2, 9], np.uint32)
    assert live_list(vis, 8).tolist() == [1, 4, 5, 7]
    assert live_list(vis, 0).tolist() == []
