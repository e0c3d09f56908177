"""The chunk generator and restatement of tests/test_gpu_chunk_numerics.py, checked without a GPU at a reduced size.

n = 3 000 store keys, 2-3 requests, Hq 8 / Hkv 2 (and G = 7): every case's named perturbations -- the causal limit +-1, the
window base off by one, the tile at a split boundary, the last split, the uncentred chunk keys (R1), the dense prefix (shared
dense), the private filter (shared spill) -- must move the fp64 output by >= 10x the bar, as the GPU file asserts before its
library calls.  The host split formula is checked against the counts the GPU file pins.
"""
import pytest
import torch

from tests.support.chunk_cases import Case, host_splits, split_per
from tests.support.fp64 import BAR, causal_ref, centred

SMALL = dict(n=3000, p=3000, Hq=8, Hkv=2, dev="cpu")


@pytest.mark.parametrize("regime,place", [("R1", None), ("R2", None), ("R4", "split_start"), ("R4", "split_end"),
                                          ("R4", "own_row")], ids=["R1", "R2", "R4start", "R4end", "R4own"])
@pytest.mark.parametrize("T", [1, 37])
def test_chunk_regime_is_sensitive(regime, place, T):
    c = Case(regime, 2, T, place=place or "split_start", seed=5 + T, sms=8, **SMALL)
    for layer in ("sparse", "dense"):
        names = set(c.perturbations(layer))
        assert ("sees_next_row" in names) == (T > 1) and ("uncentred_chunk_keys" in names) == (regime == "R1" and layer == "sparse")
        _, moved = c.check_inputs(layer)
        assert set(moved) == names


@pytest.mark.parametrize("regime", ["R1", "R2", "R4"])
def test_shared_spill_is_sensitive(regime):
    """Three requests on one slot, each with spilled keys of its own: seeing every request's, or none of its own, moves every
    request."""
    c = Case(regime, 3, 16, C=1, spill=True, x=(40, 67, 101), seed=11, sms=132, **SMALL)
    assert [hi - lo for _, lo, hi in c.priv[0]] == [40, 67, 101]
    assert all(w.shape[1] == 4 + 64 for w in c.win_k)
    _, moved = c.check_inputs("sparse")
    assert {"sees_all_private", "sees_no_private"} <= set(moved)


def test_shared_dense_prefix_is_sensitive():
    c = Case("R2", 2, 37, Hq=28, Hkv=4, n=3000, p=3000, C=1, tail=True, seed=13, sms=132, dev="cpu")
    _, moved = c.check_inputs("dense")
    assert "no_dense_prefix" in moved


def test_stale_lengths_is_sensitive():
    """The capture case's check after a spill: the restatement over the store length before the spill must differ."""
    c = Case("R1", 1, 16, seed=17, sms=132, **SMALL)
    c.commit([16])
    c.stale_n = [k.shape[1] for k in c.store_k]
    c.do_spill()
    _, moved = c.check_inputs("sparse", capture=True)
    assert "stale_lengths" in moved


def test_host_split_formula():
    """The (m-blocks, splits) the GPU file pins for the chunk line's shapes on 132 SMs, and the split edges it relies on."""
    keys = 97932 + 68
    assert host_splits(64, 4, 8, 1, 132, keys + 64) == (2, 16)
    assert host_splits(256, 4, 8, 1, 132, keys + 256) == (8, 4)
    assert host_splits(1024, 4, 8, 1, 132, keys + 1024) == (32, 1)
    assert host_splits(64, 4, 8, 8, 132, keys + 64) == (2, 2)
    # dense, Hq 8 / Hkv 1, prefix 600, T = 1024: m-block 0 (tokens 0-15) ends before the third split begins
    nmb, sp = host_splits(1024, 8, 1, 1, 132, 600 + 1024)
    assert (nmb, sp) == (64, 3) and (sp - 1) * split_per(1624, sp) >= 600 + 16


def test_restatement_matches_causal_ref():
    """The combined-axis restatement equals causal_ref (store + window before the chunk, the chunk causal)."""
    c = Case("R1", 1, 9, Hq=4, Hkv=1, n=300, p=200, seed=19, sms=132, dev="cpu")
    o = c.restate("sparse")
    ctx_k = torch.cat([c.store_k[0][0], c.win_k[0][0]])
    ctx_v = torch.cat([c.store_v[0][0], c.win_v[0][0]])
    ref = causal_ref(c.q[0], ctx_k, ctx_v, centred(c.k[0, :, 0], c.avg[0][0]), c.v[0, :, 0])
    assert torch.allclose(o[0], ref, atol=1e-12)
    ref = causal_ref(c.q[0], c.dk[0][:, 0], c.dv[0][:, 0], c.k[0, :, 0], c.v[0, :, 0])
    assert torch.allclose(c.restate("dense")[0], ref, atol=1e-12)
    assert BAR == 1e-3
