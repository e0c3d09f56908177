"""The model-shaped input regimes of tests/test_gpu_numerics.py, checked without a GPU.

Each regime's generator must produce inputs on which its property holds (R2: the window holds >= 90 % of the mass, R3: a
window share in [0.3, 0.7], R4: scores spanning >= 40 nats, R5: a sampled key past cos = 1) and on which the named perturbation
of the fp64 restatement moves the output by >= 10x the 1e-3 bar.  Codes come from the CPU-side hashing (synth.hash_keys for the
keys, the C oracle's SimHash for the queries), so a regime that has gone insensitive fails here first.
"""
import math

import pytest
import torch

from tests.support.fp64 import BAR, merge2, restate, softmax_state
from tests.support.sparse_cases import TREE, check_case, check_dense, cpu_codes, make_case, make_dense

REGIMES = [("R1", "last"), ("R2", "last"), ("R3", "last"), ("R4", "first"), ("R4", "last"), ("R5", "last")]


@pytest.mark.parametrize("regime,place", REGIMES, ids=["R1", "R2", "R3", "R4f", "R4l", "R5"])
def test_sparse_regime_is_sensitive(regime, place):
    c = make_case(regime, 1, 8, 2, 1500, 8, 40, seed=3, place=place)
    check_case(c)


@pytest.mark.parametrize("regime", ["R1", "R2", "R3", "R4"])
def test_tree_regime_is_sensitive(regime):
    parents = [TREE] * 2
    c = make_case(regime, 2, 4, 1, 800, 7, 30, seed=4, T=8, parents=parents)
    check_case(c, parents)


@pytest.mark.parametrize("P,place", [(1, "new"), (31, "first"), (33, "last"), (300, "first")])
@pytest.mark.parametrize("regime", ["R2", "R4"])
def test_dense_regime_is_sensitive(regime, P, place):
    check_dense(make_dense(regime, 2, 8, 2, P, 1, seed=P, place=place))
    check_dense(make_dense(regime, 1, 8, 2, P, 4, seed=P + 1, place=place, one_prompt=True))


def test_restatement_pieces():
    """The restatement's pieces on cases with a known answer."""
    g = torch.Generator().manual_seed(0)
    z = torch.randn(100, generator=g, dtype=torch.float64) * 3
    v = torch.randn((100, 8), generator=g, dtype=torch.float64)
    o, lse = softmax_state(z, v)
    p = torch.softmax(z, 0)
    assert torch.allclose(o, p @ v, rtol=0, atol=1e-12)
    assert abs(lse - float(torch.logsumexp(z, 0)) / math.log(2)) < 1e-12
    # split in two and merged by base-2 LSE = the whole; the tiled form with every rescale = the whole too
    oa, la = softmax_state(z[:37], v[:37])
    ob, lb = softmax_state(z[37:], v[37:])
    assert torch.allclose(merge2(oa, la, ob, lb), o, rtol=0, atol=1e-12)
    assert not torch.allclose(merge2(oa, la, ob, lb, natural=True), o, rtol=0, atol=1e-9)
    # clamp: a key exactly along q with a norm rounded down gets the weight of cos = 1, not NaN
    c = make_case("R5", 1, 4, 1, 400, 6, 20, seed=1)
    out, _, _ = restate(c, cpu_codes(c))
    assert torch.isfinite(out).all()
    assert BAR == 1e-3
