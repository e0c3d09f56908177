"""The batched generator and restatement of tests/test_gpu_batch_numerics.py, checked without a GPU at a reduced size.

n = 3 000 keys per slot, four requests on two slots holding different documents, ragged windows: each regime's property must
hold (R2: the window holds >= 90 % of the mass, R4: scores spanning >= 40 nats) and every named perturbation -- the regime's
own, `window_of_request_0` and `wrong_document` -- must move the fp64 output by >= 10x the 1e-3 bar.  The dense generator
(one prompt, ragged tails) likewise.
"""
import pytest
import torch

from magicpig_b200 import synth
from tests.support.fp64 import key_codes, query_codes
from tests.support.sparse_cases import LENS, TREE, check_dense_inputs, check_inputs, make_batch, make_dense_slots, perturbations

SMALL = dict(n=3000, dev="cpu", Hq=8, Hkv=2, K=8, L=60)


@pytest.mark.parametrize("regime,place", [("R1", "key"), ("R2", "key"), ("R4", "key"), ("R4", "win")],
                         ids=["R1", "R2", "R4key", "R4win"])
def test_batch_regime_is_sensitive(regime, place):
    c = make_batch(regime, 4, C=2, place=place, seed=7, **SMALL)
    assert len({w.shape[1] for w in c["win_k"]}) == len(set(LENS)), "windows are not ragged"
    assert set(perturbations(c)) >= ({"window_of_request_0", "wrong_document"} if regime != "R2" and place == "key" else {"window_of_request_0"})
    moved = check_inputs(c)
    assert set(moved) == set(perturbations(c))


def test_tree_batch_is_sensitive():
    parents = [TREE] * 2
    c = make_batch("R2", 2, C=1, T=8, lens=(69, 150), seed=8, parents=parents, **SMALL)
    check_inputs(c, parents)


@pytest.mark.parametrize("regime", ["R2", "R4"])
def test_dense_slots_is_sensitive(regime):
    c = make_dense_slots(regime, 4, 500, 4, seed=9, dev="cpu", Hq=8, Hkv=2)
    assert len({t[0].shape[0] for t in c["tails"]}) > 1, "tails are not ragged"
    check_dense_inputs(c)


def test_codes_match_the_packing():
    """The fp64 key codes pack as synth.hash_keys; the query codes are the reference's normalisation and projection."""
    hf = synth.make_hash_func(128, 6, 20, seed=2)
    g = torch.Generator().manual_seed(1)
    key = torch.randn((2, 700, 128), generator=g).bfloat16()
    ours, ref = key_codes(key, hf, 6, 20), synth.hash_keys(key, hf, 6, 20)
    assert (ours != ref).float().mean() < 1e-3     # fp32 against fp64 accumulation: only projections near zero differ
    q = torch.randn((3, 128), generator=g).bfloat16()
    codes, margin = query_codes(q, hf, 6, 20)
    ref = synth.hash_queries_ref(q, hf, 6, 20)
    bad = codes != ref
    assert not bool(bad.any()) or float(margin[bad].max()) < 1e-4
