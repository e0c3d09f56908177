"""Chunk steps on the host: the turn planner of LlamaDecodeRunner.extend() and the fp64 reference tests/test_gpu_chunk.py uses
(support.fp64.causal_ref)."""
import math

import pytest
import torch

from magicpig_b200.llama_runner import plan_turn_chunks
from tests.support.chunk_cases import Case
from tests.support.fp64 import BAR, causal_ref, rel_rows


def test_plan_turn_chunks_ragged():
    plan = plan_turn_chunks([300, 250, 0], t_max=256, room=128)
    assert [(s, T) for s, T, _ in plan] == [(0, 128), (128, 128), (256, 44)]
    assert plan[0][2] == [0, 0, 128] and plan[1][2] == [0, 6, 128] and plan[2][2] == [0, 44, 44]
    # every request keeps exactly its length over the turn
    for b, n in enumerate([300, 250, 0]):
        assert sum(T - drop[b] for _, T, drop in plan) == n


@pytest.mark.parametrize("t_max,room", [(1024, 192), (64, 1000), (1, 5)])
def test_plan_turn_chunks_bounds(t_max, room):
    lengths = [1, 777, 512]
    plan = plan_turn_chunks(lengths, t_max, room)
    assert all(1 <= T <= min(t_max, room) for _, T, _ in plan)
    assert len(plan) == math.ceil(max(lengths) / min(t_max, room))
    assert [s for s, _, _ in plan] == [i * min(t_max, room) for i in range(len(plan))]
    for b, n in enumerate(lengths):
        assert sum(T - drop[b] for _, T, drop in plan) == n
        assert all(0 <= drop[b] <= T for _, T, drop in plan)


def test_plan_turn_chunks_refuses():
    assert plan_turn_chunks([0, 0], 8, 8) == []
    with pytest.raises(ValueError):
        plan_turn_chunks([3], 0, 8)
    with pytest.raises(ValueError):
        plan_turn_chunks([-1], 8, 8)


def test_causal_ref_matches_naive_loop():
    g = torch.Generator().manual_seed(3)
    T, G, d, n = 5, 3, 16, 7
    q, kc, vc = torch.randn((T, G, d), generator=g), torch.randn((T, d), generator=g), torch.randn((T, d), generator=g)
    kx, vx = torch.randn((n, d), generator=g), torch.randn((n, d), generator=g)
    out = causal_ref(q, kx, vx, kc, vc)
    for t in range(T):
        for j in range(G):
            keys = [kx[i] for i in range(n)] + [kc[i] for i in range(t + 1)]
            vals = [vx[i] for i in range(n)] + [vc[i] for i in range(t + 1)]
            s = [float(q[t, j].double() @ k.double()) / math.sqrt(d) for k in keys]
            m = max(s)
            w = [math.exp(x - m) for x in s]
            o = sum(wi * v.double() for wi, v in zip(w, vals)) / sum(w)
            assert torch.allclose(out[t, j], o, atol=1e-12)


def _chunk_kernel_emulation(q, K, V, split, splits=1, lim=None, keep=None):
    """The chunk kernel's arithmetic for one kv-group: 64-key tiles, online softmax in fp32 (log2 units), P = exp2(s - m) in fp32,
    l summed from that P, and P entering P.V either rounded to bf16 (split = False) or as bf16 hi + bf16 lo (split = True).
    splits > 1: the key axis cut as launch_chunk_attend cuts it (equal ranges of whole 64-key tiles), each split's state (m in
    natural-log units, l, acc) kept in fp32 and merged as merge_states merges them.  lim (R,): the last key each row sees (the
    causal limit); keep (n,): the private filter."""
    bf = lambda x: x.bfloat16().float()   # noqa: E731
    R, d = q.shape
    n = K.shape[0]
    dev = q.device
    lim = torch.full((R,), n - 1, device=dev) if lim is None else lim
    keep = torch.ones(n, dtype=torch.bool, device=dev) if keep is None else keep
    c = 1.4426950408889634 / math.sqrt(d)
    per = ((n + splits - 1) // splits + 63) // 64 * 64
    states = []
    for sp in range(splits):
        m, l, acc = torch.full((R,), -math.inf, device=dev), torch.zeros(R, device=dev), torch.zeros(R, d, device=dev)
        end = min(sp * per + per, n)
        for k0 in range(sp * per, end, 64):
            k1 = min(k0 + 64, end)
            s = (q @ K[k0:k1].T) * c
            vis = (torch.arange(k0, k1, device=dev)[None] <= lim[:, None]) & keep[None, k0:k1]
            s = torch.where(vis, s, torch.tensor(-math.inf, device=dev))
            mn = torch.maximum(m, s.max(1).values)
            muse = torch.where(mn == -math.inf, torch.zeros(R, device=dev), mn)   # a row with no visible key yet: all p = 0
            corr = torch.where(m == -math.inf, torch.zeros(R, device=dev), torch.exp2(m - mn))
            p = torch.exp2(s - muse[:, None])
            l, acc = l * corr + p.sum(1), acc * corr[:, None]
            ph = bf(p)
            acc = acc + ph @ V[k0:k1]
            if split:
                acc = acc + bf(p - ph) @ V[k0:k1]
            m = mn
        states.append((m * 0.6931471805599453, l, acc))
    if splits == 1:
        return acc / l[:, None]
    ms = torch.stack([s_[0] for s_ in states])
    M = ms.max(0).values
    f = torch.where(ms == -math.inf, torch.zeros((), device=dev), torch.exp2((ms - M) * 1.4426950408889634))
    L = sum(f[i] * states[i][1] for i in range(splits))
    A = sum(f[i][:, None] * states[i][2] for i in range(splits))
    return A / L[:, None]


def test_p_split_is_needed_for_the_1e3_bar():
    """Why P enters P.V as bf16 hi + lo: with queries 4x the usual scale (logit std 4, a few keys take most of the probability) over
    20 000 keys, plain bf16 P misses 1e-3 of fp64; the split stays ~1e-5.  (At unit scale both pass.)"""
    g = torch.Generator().manual_seed(0)
    n, d = 20000, 128
    K = torch.randn((n, d), generator=g).bfloat16().float()
    V = torch.randn((n, d), generator=g).bfloat16().float()
    q = (torch.randn((128, d), generator=g) * 4).bfloat16().float()
    ref = torch.softmax(q.double() @ K.double().T / math.sqrt(d), 1) @ V.double()
    plain = (_chunk_kernel_emulation(q, K, V, False).double() - ref).abs().max().item()
    split = (_chunk_kernel_emulation(q, K, V, True).double() - ref).abs().max().item()
    assert plain > 1e-3, plain
    assert split < 1e-4, split


@pytest.mark.parametrize("regime,place", [("R1", None), ("R2", None), ("R4", "split_start"), ("R4", "split_end"),
                                          ("R4", "own_row")], ids=["R1", "R2", "R4start", "R4end", "R4own"])
def test_split_merge_stays_inside_the_bar(regime, place):
    """The kernel's arithmetic over 98 000 keys cut into 16 splits and merged (a 64-token chunk of one kv-group of four heads,
    the generator of tests/test_gpu_chunk_numerics.py on the host) stays >= 10x inside the per-row relative bar of that file
    in every one of its regimes: the bar's basis."""
    c = Case(regime, 1, 32, Hq=4, Hkv=1, n=97932, p=64, place=place or "split_start", seed=3, dev="cpu",
             check_layers=("sparse",))
    sp = c.splits("sparse")
    assert sp == 16
    K, V, keep, nA, jb0 = c.axis(0, "sparse")
    lim = (nA + jb0 + torch.arange(c.T)).repeat_interleave(c.G)
    q = c.q[0].reshape(-1, c.q.shape[-1]).float()
    got = _chunk_kernel_emulation(q, K[0].float(), V[0].float(), True, splits=sp, lim=lim, keep=keep)
    err = rel_rows(got, c.restate("sparse")[0].reshape(got.shape))
    assert err <= BAR / 10, f"{regime}: {err:.2e}"
