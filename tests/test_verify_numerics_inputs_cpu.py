"""The generators and self-checks of tests/test_gpu_verify_numerics.py without a GPU, at a reduced size: n = 3 000 stored keys,
K8 L60, Hq 32 / Hkv 8, a window of NS + NL filled rows, a dense prompt of 2 000 rows.

Every (step, regime) pair of the GPU file must keep its regime's property and have its perturbations move the fp64 output by
>= 10x the 1e-3 bar: the regime's own, `tree_as_chain` for the R2 trees, and for the steps after each accept or rewind the wrong
commits (`node_order`, `path_dropped`, `step_kept`) that differ from the right one.  Run with -s to see how far each moves the
output.
"""
import pytest
import torch

from tests.support.fp64 import BAR, centred, rel_rows
from tests.support.library import NL, NS
from tests.support.sparse_cases import (ACCEPT_IDS, ACCEPTS, ACCEPT_VARIANTS, GEN, LINE_TREES, check_after, check_dense_after,
                                        check_inputs, committed_as, dense_moves, make_batch, make_dense, next_case,
                                        next_dense)

SMALL = dict(n=3000, dev="cpu", Hq=32, Hkv=8, K=8, L=60)
P, W = 2000, NS + NL
_BASE = {}


def sparse_inputs(regime, T, parents=None, place="key", lens=None, seed=0):
    if regime not in _BASE:
        _BASE[regime] = make_batch(regime, 1, lens=(NS + 8,), place="win", seed=3, **SMALL)
    return make_batch(regime, 1, T=T, lens=lens or (W + T,), place=place, seed=seed, parents=parents, base=_BASE[regime],
                      **SMALL)


def show(label, moved):
    print(f"{label}: " + ", ".join(f"{k} {v:.2e}" for k, v in moved.items()))
    assert min(moved.values()) >= 10 * BAR


SPARSE = ([(f"T{T} {r}", r, T, None, "key", None) for T in (2, 4, 8) for r in ("R1", "R2", "R4")]
          + [("T8 R2 full window", "R2", 8, None, "key", NS + NL + GEN)]
          + [(f"{t} {r}", r, len(LINE_TREES[t]), t, p, None) for t in LINE_TREES for r, p in (("R2", "key"), ("R4", "win"))])


@pytest.mark.parametrize("label,regime,T,tree,place,rows", SPARSE, ids=[s[0].replace(" ", "-") for s in SPARSE])
def test_sparse_inputs(label, regime, T, tree, place, rows):
    parents = None if tree is None else [LINE_TREES[tree]]
    c = sparse_inputs(regime, T, parents, place, None if rows is None else (rows,), seed=T)
    extra = ("tree_as_chain",) if tree and regime == "R2" else ()
    moved = check_inputs(c, parents, extra=extra)
    assert set(extra) <= set(moved)
    show(label, moved)


DENSE = ([(f"T{T} {r}{p}", r, T, None, p) for T in (2, 4, 5, 6, 7, 8) for r, p in (("R2", ""), ("R4", "first"), ("R4", "last"),
                                                                                       ("R4", "new"))]
         + [(f"{t} R2", "R2", len(LINE_TREES[t]), t, "") for t in LINE_TREES])


@pytest.mark.parametrize("label,regime,T,tree,place", DENSE, ids=[s[0].replace(" ", "-") for s in DENSE])
def test_dense_inputs(label, regime, T, tree, place):
    parents = None if tree is None else [LINE_TREES[tree]]
    dn = make_dense(regime, 1, 32, 8, P, T, seed=T, place=place or "last")
    o, moved = dense_moves(dn, parents, ("tree_as_chain",) if tree else ())
    assert torch.isfinite(o).all()
    show(f"dense {label}", moved)


@pytest.mark.parametrize("label,tree,path", ACCEPTS, ids=ACCEPT_IDS)
def test_accept_inputs(label, tree, path):
    """The step and the two that follow its accept or rewind, sparse and dense: every wrong commit that differs from the right
    one moves both following steps."""
    T = 8 if tree is None else len(tree)
    parents = None if tree is None else [tree]
    c = sparse_inputs("R2", T, parents, seed=20 + T)
    dn = make_dense("R2", 1, 32, 8, P, T, seed=30 + T)
    extra = ("tree_as_chain",) if tree else ()
    show(f"{label} step", check_inputs(c, parents, extra=extra))
    show(f"{label} step dense", dense_moves(dn, parents, extra)[1])
    wrong = {v for v in ACCEPT_VARIANTS if committed_as(v, [path], T) != [path]}
    assert wrong == ({"step_kept"} if not path else {"path_dropped", "step_kept"} | ({"node_order"} if tree else set()))
    for fn, case, name in ((check_after, c, "sparse"), (check_dense_after, dn, "dense")):
        cases, moved = fn(case, [path], (1, 2), seed=40)
        assert wrong <= set(moved) and [x["q"].shape[1] for x in cases] == [1, 2]
        show(f"{label} next {name}", moved)


def test_next_case_commits_in_path_order():
    """next_case appends the committed rows' keys centred (fp32 subtraction, one bf16 rounding) and their values, in the order
    given; next_dense appends the raw rows; neither draw depends on what was committed."""
    c = sparse_inputs("R2", 7, [LINE_TREES["binary_depth3"]], seed=5)
    a, b = next_case(c, [[0, 2, 5]], 2, seed=1), next_case(c, [[]], 2, seed=1)
    assert a["win_k"][0].shape[1] == c["win_k"][0].shape[1] + 3 and b["win_k"][0].shape[1] == c["win_k"][0].shape[1]
    tail_k, tail_v = a["win_k"][0][:, -3:], a["win_v"][0][:, -3:]
    for i, t in enumerate((0, 2, 5)):
        assert torch.equal(tail_k[:, i], centred(c["k_new"][0, t], c["slots"][0]["avg"]))
        assert torch.equal(tail_v[:, i], c["v_new"][0, t])
    assert all(torch.equal(a[k], b[k]) for k in ("q", "k_new", "v_new"))
    dn = make_dense("R2", 1, 32, 8, 100, 8, seed=6)
    x, y = next_dense(dn, [[0, 7]], 1, seed=2), next_dense(dn, [[0, 1]], 1, seed=2)
    assert x["P"] == 102 and torch.equal(x["dk"][0, 100:], dn["k"][0, [0, 7]]) and torch.equal(x["dv"][0, 100:], dn["v"][0, [0, 7]])
    assert all(torch.equal(x[k], y[k]) for k in ("q", "k", "v"))
    assert rel_rows(x["dk"][0, 101].float(), y["dk"][0, 101].float()) > 0
