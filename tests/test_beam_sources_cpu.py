"""beam_sources: the map a beam-search step hands to reorder(), checked on the CPU.

For new beams with parents p (new beam i continues old beam p[i], held by request p[i]), beam_sources returns request_of (where
new beam i lives) and src_of (the reorder map).  What the reorder kernel relies on, and what the caller relies on:
  - every source is a fixed point: src_of[src_of[b]] == src_of[b] (no request is both read and written);
  - src_of[request_of[i]] == parents[i] (each new beam continues its parent's sequence);
  - request_of is a permutation (every new beam has a request of its own);
plus the placement rule: a parent's first child stays in the parent's request, later children take the unchosen parents'
requests in ascending order.
"""
import random

import pytest
import torch

from magicpig_b200.attnserver import beam_sources


def check(parents):
    p = torch.as_tensor(parents, dtype=torch.int64)
    B = p.numel()
    src_of, request_of = beam_sources(p)
    assert src_of.dtype == torch.int32 and request_of.dtype == torch.int32
    assert tuple(src_of.shape) == (B,) and tuple(request_of.shape) == (B,)
    s, r, pl = src_of.tolist(), request_of.tolist(), p.tolist()
    assert all(0 <= x < B for x in s)
    assert all(s[s[b]] == s[b] for b in range(B)), (pl, s)
    assert sorted(r) == list(range(B)), (pl, r)
    assert all(s[r[i]] == pl[i] for i in range(B)), (pl, s, r)
    # the placement rule, restated on the host
    seen, free = set(), iter(sorted(set(range(B)) - set(pl)))
    want = []
    for i, q in enumerate(pl):
        want.append(q if q not in seen else next(free))
        seen.add(q)
    assert r == want, (pl, r, want)
    # requests nobody moves into keep their sequence
    assert all(s[b] == b for b in set(pl))


@pytest.mark.parametrize("B", list(range(1, 33)))
def test_adversarial(B):
    check([0] * B)                       # every beam from one parent (the first step from a prompt)
    check([B - 1] * B)                   # ... from the last one
    check(list(range(B)))                # the identity: nothing moves
    check(list(reversed(range(B))))      # a permutation: every beam survives, each in its own request
    rng = random.Random(B)
    perm = list(range(B))
    rng.shuffle(perm)
    check(perm)
    check([i // 2 * 2 for i in range(B)])          # pairs: every even beam twice
    check(sorted(rng.randrange(B) for _ in range(B)))


@pytest.mark.parametrize("seed", range(50))
def test_random(seed):
    rng = random.Random(1000 + seed)
    B = rng.randint(1, 32)
    k = rng.randint(1, B)                # parents drawn from k of the beams
    pool = rng.sample(range(B), k)
    check([rng.choice(pool) for _ in range(B)])


def test_traceable_shapes():
    """No data-dependent shapes: the outputs have B entries whatever the parents (what a CUDA graph needs)."""
    for parents in ([3, 3, 3, 3], [0, 1, 2, 3], [2, 0, 2, 1]):
        src_of, request_of = beam_sources(torch.tensor(parents))
        assert src_of.shape == request_of.shape == (4,)
