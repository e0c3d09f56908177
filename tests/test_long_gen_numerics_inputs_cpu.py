"""The generators, host mirrors and self-checks of tests/test_gpu_long_gen_numerics.py without a GPU: the full-size schedule and
partition (pure Python), and the dense tails, their fp64 restatements and perturbations at a reduced size (a 300-row prompt,
tails of several 32-row tiles)."""
import pytest
import torch

from tests.support.library import NL, NS
from tests.support.fp64 import rel_rows
from tests.support.long_gen import DenseTails, PrivateRuns, check_dense_tails, restate_chunk, schedule, tail_items
from tests.support.sparse_cases import GEN, HKV, HQ, M_LONG, N_C2, TREE

TAILS = (4096, 4095, 4097, 4128, 4127, 4392, 4064, 4100)
SMALL = (128, 127, 129, 160, 96, 152, 100, 159)


def _events(tails, chunk_at=(2000, 3500), t_chunk=40):
    return schedule(tails, 4, NS, NS + NL + GEN, NL - 16, chunk_at, t_chunk)


def test_full_schedule():
    """The shared line's schedule: 16 spills, every request spilling at each, the private keys within max_length, every
    window with room for the 8-node tree at the end, two chunk steps over tails of thousands of rows."""
    ev, w = _events(TAILS)
    spills = [g for kind, g in ev if kind == "spill"]
    assert len(spills) == 16 and all(min(g) > 0 for g in spills)
    assert N_C2 + sum(map(sum, spills)) <= M_LONG
    assert max(w) + 8 <= NS + NL + GEN
    done, chunks = [0] * 8, []
    for kind, x in ev:
        if kind == "chunk":
            chunks.append(min(done))
        if kind != "spill":
            done = [dn + (40 if kind == "chunk" else 4) - dr for dn, dr in zip(done, x)]
    assert done == list(TAILS) and len(chunks) == 2 and min(chunks) >= 1900
    runs = PrivateRuns(8, N_C2)
    for g in spills:
        runs.spill(g)
    assert runs.total == N_C2 + sum(map(sum, spills)) and all(len(r) == 16 for r in runs.runs)


def test_full_partition():
    """On a 132-SM H100 the T = 1 step over the line's tails has items inside a tail and items starting inside one; a short
    tail has neither."""
    inside, boundary = tail_items(98000, [t + 1 for t in TAILS], 1, HQ // HKV, HKV, 132 * 8)
    assert inside >= 1 and boundary >= 1
    assert tail_items(98000, [17] * 8, 1, HQ // HKV, HKV, 132 * 8) == (0, 0)


def test_private_runs_visibility_and_fork():
    runs = PrivateRuns(3, 10)
    runs.spill([2, 0, 3])
    runs.spill([1, 2, 1])
    assert runs.runs == [[(10, 12), (15, 16)], [(16, 18)], [(12, 15), (18, 19)]]
    assert runs.visibility(12, "cpu")[:9].tolist() == [1, 1, 4, 4, 4, 1, 2, 2, 4]
    runs.fork(2, 0)
    assert runs.visibility(12, "cpu")[:9].tolist() == [0, 0, 5, 5, 5, 0, 2, 2, 5]
    m = runs.masks(runs.runs, "cpu")
    assert m[0].tolist() == [True] * 10 + [False, False, True, True, True, False, False, False, True]


@pytest.fixture(scope="module")
def small():
    """A reduced shared-prefix dense layer: P = 300, B = 8 on one slot, tails of 96..160 rows from the schedule's T-token steps
    and one chunk step (checked against its restatement without the tail)."""
    dt = DenseTails(8, 300, 176, HKV, [40 + 5 * b for b in range(8)], 7, "cpu")
    ev, _ = schedule(SMALL, 4, NS, NS + NL + 60, NL - 16, (60,), 16)
    moved = []
    for kind, x in ev:
        if kind == "spill":
            continue
        n = 4 if kind == "step" else 16
        keep = [n - dr for dr in x]
        k, v = dt.step_rows(n, keep)
        if kind == "chunk":
            q = dt.check_step("R2", n, HQ)[0]
            moved.append(rel_rows(restate_chunk(dt, q, k, v, "ignores_tail"), restate_chunk(dt, q, k, v)))
        dt.commit(k, v, keep)
    assert dt.tl == list(SMALL)
    return dt, moved


def test_small_chunk_sees_tail(small):
    _, moved = small
    assert len(moved) == 1 and moved[0] >= 1e-2


@pytest.mark.parametrize("regime", ["R2", "R4"])
@pytest.mark.parametrize("shape", ["T1", "T4", "tree8"])
def test_small_dense_self_checks(small, shape, regime):
    dt, _ = small
    T = {"T1": 1, "T4": 4, "tree8": 8}[shape]
    q, k, v = dt.check_step(regime, T, HQ)
    o, moved = check_dense_tails(dt, regime, q, k, v, [TREE] * 8 if shape == "tree8" else None)
    assert torch.isfinite(o).all()
    assert ("sees_previous_member_tail" in moved) == (shape != "tree8")


def test_small_partition(small):
    """At the reduced size every group's items are a tile or two long, so items lie inside tails and start inside them."""
    dt, _ = small
    inside, boundary = tail_items(dt.P, [t + 1 for t in dt.tl], 1, HQ // HKV, HKV, 132 * 8)
    assert inside >= 8 and boundary >= 8
