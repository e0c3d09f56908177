"""Token-tree verification steps (`-m gpu`): mpig_plan_tree -> mpig_decode_tokens / mpig_dense_decode_tokens -> mpig_accept.

Node t of a tree step must equal a chain step over its root path:
  * sparse layers: identical query codes, nnz and index lists, fp32 outputs within 1e-5, each node within 1e-3 of the oracle fed
    the window plus its ancestors' rows;
  * dense layers: within 1e-5 of the path chains and 1e-3 of an fp64 masked restatement;
  * a chain tree is bitwise plan_tokens; accept(path) leaves the state of a twin that ran the path as a chain step; a captured
    plan_tree -> layers -> accept replays with new trees and paths; tree steps run into a spill; refusals change nothing.
"""
import random

import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200 import synth
from tests.support.fp64 import assert_1e3_f32, assert_rounded_half_up, oracle_decode, rel_max
from tests.support.library import Run, Twins, _Cfg, assert_tables_equal, lsh_tables

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
d, NS, NL = 128, 4, 64


def random_tree(T, rng):
    return [-1] + [rng.randrange(t) for t in range(1, T)]


def root_path(par, t):
    path = [t]
    while par[path[-1]] >= 0:
        path.append(par[path[-1]])
    return path[::-1]


def twins(B, Hq, Hkv, n, K, L, T, seed, **kw):
    """Twins whose `seq` context also takes steps of up to T tokens: the reference that runs root paths as chain steps."""
    tw = Twins(B, Hq, Hkv, n, K, L, T, seed, **kw)
    tw.seq.reserve_query_tokens(T)
    return tw


def readout(ctx, B, T, Hq, sparse=True):
    r = dict(o32=ctx.last_out_f32().cpu().reshape(B, T, Hq, d))
    if sparse:
        nnz, res = ctx.last_probe(want_results=True)
        r.update(nnz=nnz.cpu().reshape(B, T, Hq), res=res.cpu().reshape(B, T, Hq, -1),
                 codes=ctx.last_codes().cpu().reshape(B, T, Hq, -1))
    return r


def tree_step(ctx, pars, q, k, v, layers=(1,)):
    """plan_tree + the layers; returns {layer: (out, readout)}."""
    B, T, Hq = q.shape[0], q.shape[1], q.shape[2]
    ctx.plan(T, parents=torch.tensor(pars, dtype=torch.int32, device=DEV))
    got = {}
    for layer in layers:
        fn = ctx.decode_tokens if layer == 1 else ctx.dense_decode_tokens
        out = fn(layer, T, q.to(DEV), k.to(DEV), v.to(DEV)).cpu().reshape(B, T, Hq, d)
        got[layer] = (out, readout(ctx, B, T, Hq, layer == 1))
    return got


def path_chains(ctx, pars, q, k, v, layers=(1,)):
    """For every node t: a chain step over each request's root path of t (padded to the longest path), read at the path's end,
    then rewound.  Returns {layer: readout (B, T, Hq, ...)} in node order."""
    B, T, Hq = q.shape[0], q.shape[1], q.shape[2]
    per = {layer: [] for layer in layers}
    for t in range(T):
        paths = [root_path(pars[b], t) for b in range(B)]
        P = max(len(p) for p in paths)
        idx = torch.tensor([p + [p[-1]] * (P - len(p)) for p in paths])
        gather = lambda x: torch.stack([x[b, idx[b]] for b in range(B)]).contiguous()
        qc, kc, vc = gather(q), gather(k), gather(v)
        ctx.plan(P)
        for layer in layers:
            fn = ctx.decode_tokens if layer == 1 else ctx.dense_decode_tokens
            fn(layer, P, qc.to(DEV), kc.to(DEV), vc.to(DEV))
            r = readout(ctx, B, P, Hq, layer == 1)
            per[layer].append({key: torch.stack([x[b, len(paths[b]) - 1] for b in range(B)]) for key, x in r.items()})
        ctx.rewind(torch.full((B,), P, dtype=torch.int32, device=DEV))
    return {layer: {key: torch.stack([p[key] for p in per[layer]], dim=1) for key in per[layer][0]} for layer in layers}


def assert_sparse_equal(a, s, tol=1e-5):
    assert torch.equal(a["codes"], s["codes"])
    assert torch.equal(a["nnz"], s["nnz"])
    B, T, Hq = a["nnz"].shape
    for b in range(B):
        for t in range(T):
            for h in range(Hq):
                n_ = int(a["nnz"][b, t, h])
                assert torch.equal(a["res"][b, t, h, :n_], s["res"][b, t, h, :n_]), (b, t, h)
    assert rel_max(a["o32"], s["o32"]) <= tol


def test_chain_tree_equals_plan_tokens(cuda_lib):
    """plan_tree with chain parents is bitwise plan_tokens: outputs, fp32 copies, codes, nnz and index lists, both layers."""
    B, Hq, Hkv, T = 2, 8, 2, 5
    tw = twins(B, Hq, Hkv, 1500, 8, 40, T, seed=11)
    q, k, v = tw.inputs(T)
    chain = [[-1] + list(range(T - 1))] * B
    a = tree_step(tw.tok, chain, q, k, v, layers=(1, 0))
    tw.seq.plan(T)
    s = {}
    for layer in (1, 0):
        fn = tw.seq.decode_tokens if layer == 1 else tw.seq.dense_decode_tokens
        out = fn(layer, T, q.to(DEV), k.to(DEV), v.to(DEV)).cpu().reshape(B, T, Hq, d)
        s[layer] = (out, readout(tw.seq, B, T, Hq, layer == 1))
    for layer in (1, 0):
        assert torch.equal(a[layer][0], s[layer][0])
        for key in a[layer][1]:
            assert torch.equal(a[layer][1][key], s[layer][1][key]), (layer, key)


@pytest.mark.parametrize("kreg", [0, 1])
@pytest.mark.parametrize("T", [3, 8])
@pytest.mark.parametrize("B,Hq,Hkv,n,K,L", [
    (2, 16, 4, 4096, 10, 150),     # clusters of 4
    (2, 4, 1, 1500, 8, 60),        # clusters of 8
    (2, 4, 1, 70000, 8, 40),       # two key segments
    (4, 32, 8, 2000, 8, 60),       # 128 heads, one CTA each (codes from the stand-alone SimHash kernel)
    (5, 32, 8, 1200, 8, 40),       # 160 heads: 512-thread CTAs in several waves
])
def test_sparse_tree_matches_paths(cuda_lib, B, Hq, Hkv, n, K, L, T, kreg):
    tw = twins(B, Hq, Hkv, n, K, L, T, seed=n + T + 7 * kreg)
    for c in tw.ctxs:
        c.set_option("fused_kreg", kreg)
    rng = random.Random(n + T)
    pars = [random_tree(T, rng) for _ in range(B)]
    q, k, v = tw.inputs(T)
    out, a = tree_step(tw.tok, pars, q, k, v)[1]
    s = path_chains(tw.seq, pars, q, k, v)[1]
    assert_sparse_equal(a, s)
    assert_rounded_half_up(out, a["o32"], "tree step")
    if n > 5000 or K >= 10:
        return   # (as in test_sparse_tokens_match_sequential: the chains themselves are checked against the oracle there)
    for b in range(B):
        tb = dict(B=1, Hq=Hq, Hkv=Hkv, d=d, K=K, L=L, n=n, M=tw.M, hash_func=tw.hf, kcodes=tw.kcodes[b:b + 1],
                  key=tw.key[b:b + 1], value=tw.value[b:b + 1], key_norm=tw.kn[b:b + 1], avg_k=tw.avg[b:b + 1])
        for t in range(T):
            anc = root_path(pars[b], t)[:-1]
            wk = torch.cat([tw.win[b][0][None]] + [k[b:b + 1, j][:, :, None] - tw.avg[b:b + 1] for j in anc], dim=2)
            wv = torch.cat([tw.win[b][1][None]] + [v[b:b + 1, j][:, :, None] for j in anc], dim=2)
            _, nz_ref, _, o_exact = oracle_decode(tb, q[b:b + 1, t][:, :, None], k[b:b + 1, t][:, :, None],
                                                  v[b:b + 1, t][:, :, None], wk, wv, tw.G)
            assert torch.equal(a["nnz"][b, t], nz_ref)
            assert_1e3_f32(a["o32"][b, t], o_exact)


@pytest.mark.parametrize("B,Hq,Hkv,P,T", [(2, 8, 2, 777, 2), (2, 8, 2, 777, 3), (2, 8, 2, 777, 4), (3, 4, 4, 31, 8),
                                          (1, 32, 8, 20000, 8)])
def test_dense_tree(cuda_lib, B, Hq, Hkv, P, T):
    """T*G = 8 (hi/lo packed), 12 and 16 (one m-tile), 32 (two m-tiles)."""
    tw = twins(B, Hq, Hkv, 64, 4, 8, T, seed=P + T, P_dense=P)
    G = Hq // Hkv
    rng = random.Random(P * T)
    pars = [random_tree(T, rng) for _ in range(B)]
    q, k, v = tw.inputs(T)
    out, a = tree_step(tw.tok, pars, q, k, v, layers=(0,))[0]
    s = path_chains(tw.seq, pars, q, k, v, layers=(0,))[0]
    assert rel_max(a["o32"], s["o32"]) <= 1e-5
    assert_rounded_half_up(out, a["o32"], "tree step")
    for b in range(B):
        for t in range(T):
            vis = root_path(pars[b], t)
            kk = torch.cat([tw.dk[b], k[b, vis]], dim=0).double()   # (P + depth + 1, Hkv, d)
            vv = torch.cat([tw.dv[b], v[b, vis]], dim=0).double()
            qt = q[b, t].double().reshape(Hkv, G, d)
            s_ = torch.einsum("kgd,nkd->kgn", qt, kk) / d ** 0.5
            ref = torch.einsum("kgn,nkd->kgd", torch.softmax(s_, dim=-1), vv).reshape(Hq, d)
            assert_1e3_f32(a["o32"][b, t], ref)


def next_steps_equal(x, y, B, Hq, Hkv, gen):
    """Steps of 1 and 2 tokens on both contexts give bitwise the same outputs, nnz and fp32 copies (both layers)."""
    for T2 in (1, 2):
        q2 = torch.randn((B, T2, Hq, d), generator=gen).bfloat16().to(DEV)
        k2 = torch.randn((B, T2, Hkv, d), generator=gen).bfloat16().to(DEV)
        v2 = torch.randn((B, T2, Hkv, d), generator=gen).bfloat16().to(DEV)
        res = []
        for c in (x, y):
            c.plan(T2)
            o_s = c.decode_tokens(1, T2, q2, k2, v2).cpu()
            r = (o_s, c.last_out_f32().cpu(), c.last_probe()[0].cpu())
            o_d = c.dense_decode_tokens(0, T2, q2, k2, v2).cpu()
            res.append(r + (o_d, c.last_out_f32().cpu()))
        for i, (p_, q_) in enumerate(zip(*res)):
            assert torch.equal(p_, q_), (T2, i)


def spilled_equal(x, y):
    """Spill both windows: the same row counts, and the spilled records and key norms are byte-equal."""
    gx, gy = x.spill_window(), y.spill_window()
    assert torch.equal(gx, gy)
    for a_, b_ in zip(x.read_cache(1), y.read_cache(1)):
        assert torch.equal(a_, b_)


def test_accept_equals_path_chain(cuda_lib):
    """After accept(path) the window records, dense rows and lengths are those of a twin that ran the path as a chain step (then
    rewound the rest): the next steps match bitwise, and so do the spilled windows.  Accept after plan_tokens equals rewind."""
    B, Hq, Hkv, T = 2, 8, 2, 6
    tw = twins(B, Hq, Hkv, 1500, 8, 40, T, seed=21)
    rng = random.Random(5)
    pars = [random_tree(T, rng) for _ in range(B)]
    q, k, v = tw.inputs(T)
    tree_step(tw.tok, pars, q, k, v, layers=(1, 0))
    paths = [root_path(pars[0], T - 1), root_path(pars[1], 0)]   # the deepest-numbered node's path, and the root alone
    cnt = [len(p) for p in paths]
    nodes = torch.tensor([p + [0] * (T - len(p)) for p in paths], dtype=torch.int32, device=DEV)
    tw.tok.accept(nodes, torch.tensor(cnt, dtype=torch.int32, device=DEV))
    Pm = max(cnt)
    idx = [p + [p[-1]] * (Pm - len(p)) for p in paths]
    qc = torch.stack([q[b, idx[b]] for b in range(B)]).contiguous()
    kc = torch.stack([k[b, idx[b]] for b in range(B)]).contiguous()
    vc = torch.stack([v[b, idx[b]] for b in range(B)]).contiguous()
    tw.seq.plan(Pm)
    tw.seq.decode_tokens(1, Pm, qc.to(DEV), kc.to(DEV), vc.to(DEV))
    tw.seq.dense_decode_tokens(0, Pm, qc.to(DEV), kc.to(DEV), vc.to(DEV))
    tw.seq.rewind(torch.tensor([Pm - c for c in cnt], dtype=torch.int32, device=DEV))
    next_steps_equal(tw.tok, tw.seq, B, Hq, Hkv, torch.Generator().manual_seed(1))
    # accept after plan_tokens = rewind(T - count)
    q, k, v = tw.inputs(4)
    tw.tok.plan(4)
    tw.seq.plan(4)
    for c in (tw.tok, tw.seq):
        c.decode_tokens(1, 4, q.to(DEV), k.to(DEV), v.to(DEV))
        c.dense_decode_tokens(0, 4, q.to(DEV), k.to(DEV), v.to(DEV))
    tw.tok.accept(torch.arange(4, dtype=torch.int32, device=DEV).repeat(B, 1), torch.tensor([3, 0], dtype=torch.int32, device=DEV))
    tw.seq.rewind(torch.tensor([1, 4], dtype=torch.int32, device=DEV))
    next_steps_equal(tw.tok, tw.seq, B, Hq, Hkv, torch.Generator().manual_seed(2))
    assert tw.tok.error_flags() == 0
    spilled_equal(tw.tok, tw.seq)


def test_tree_graph_replay(cuda_lib):
    """plan_tree -> sparse + dense layers -> accept, captured once and replayed with new trees, paths and inputs, equals an eager
    twin; a single-token step captured before stays valid."""
    B, Hq, Hkv, n, K, L, T = 2, 8, 2, 1500, 8, 40, 5
    tw = Twins(B, Hq, Hkv, n, K, L, T, seed=31, gen=96)
    eager = Twins(B, Hq, Hkv, n, K, L, T, seed=31, gen=96).tok
    ctx = tw.tok
    q_s = torch.zeros((B, T, Hq, d), dtype=torch.bfloat16, device=DEV)
    k_s = torch.zeros((B, T, Hkv, d), dtype=torch.bfloat16, device=DEV)
    v_s = torch.zeros_like(k_s)
    q1 = torch.zeros((B, 1, Hq, d), dtype=torch.bfloat16, device=DEV)
    k1 = torch.zeros((B, 1, Hkv, d), dtype=torch.bfloat16, device=DEV)
    v1 = torch.zeros_like(k1)
    par_s = torch.tensor([[-1] + list(range(T - 1))] * B, dtype=torch.int32, device=DEV)
    nodes_s = torch.zeros((B, T), dtype=torch.int32, device=DEV)
    cnt_s = torch.zeros(B, dtype=torch.int32, device=DEV)
    out_s = torch.empty((B, T, Hq * d), dtype=torch.bfloat16, device=DEV)
    out_d = torch.empty_like(out_s)
    out1 = torch.empty((B, 1, Hq * d), dtype=torch.bfloat16, device=DEV)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    g1, gT = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        ctx.plan(1)   # warm-up outside capture (plans are cached per T); count 0 leaves the lengths where they were
        ctx.decode_tokens(1, 1, q1, k1, v1, out1)
        ctx.rewind(torch.ones(B, dtype=torch.int32, device=DEV))
        ctx.plan(T, parents=par_s)
        ctx.decode_tokens(1, T, q_s, k_s, v_s, out_s)
        ctx.dense_decode_tokens(0, T, q_s, k_s, v_s, out_d)
        ctx.accept(nodes_s, cnt_s)
        with torch.cuda.graph(g1, stream=st):
            ctx.plan(1)
            ctx.decode_tokens(1, 1, q1, k1, v1, out1)
        with torch.cuda.graph(gT, stream=st):
            ctx.plan(T, parents=par_s)
            ctx.decode_tokens(1, T, q_s, k_s, v_s, out_s)
            ctx.dense_decode_tokens(0, T, q_s, k_s, v_s, out_d)
            ctx.accept(nodes_s, cnt_s)
    torch.cuda.current_stream().wait_stream(st)
    torch.cuda.synchronize()
    rng = random.Random(3)
    for it in range(4):
        pars = [random_tree(T, rng) for _ in range(B)]
        paths = [root_path(p, rng.randrange(T)) for p in pars]
        nodes = torch.tensor([p + [0] * (T - len(p)) for p in paths], dtype=torch.int32)
        cnt = torch.tensor([len(p) for p in paths], dtype=torch.int32)
        q, k, v = tw.inputs(T)
        q_s.copy_(q), k_s.copy_(k), v_s.copy_(v)
        par_s.copy_(torch.tensor(pars, dtype=torch.int32))
        nodes_s.copy_(nodes), cnt_s.copy_(cnt)
        gT.replay()
        torch.cuda.synchronize()
        eager.plan(T, parents=torch.tensor(pars, dtype=torch.int32, device=DEV))
        e_s = eager.decode_tokens(1, T, q.to(DEV), k.to(DEV), v.to(DEV)).cpu()
        e_d = eager.dense_decode_tokens(0, T, q.to(DEV), k.to(DEV), v.to(DEV)).cpu()
        eager.accept(nodes.to(DEV), cnt.to(DEV))
        assert torch.equal(out_s.cpu(), e_s), it
        assert torch.equal(out_d.cpu(), e_d), it
        qq, kk, vv = tw.inputs(1)
        q1.copy_(qq), k1.copy_(kk), v1.copy_(vv)
        g1.replay()
        torch.cuda.synchronize()
        eager.plan(1)
        e1 = eager.decode_tokens(1, 1, qq.to(DEV), kk.to(DEV), vv.to(DEV)).cpu()
        assert torch.equal(out1.cpu(), e1), it
    assert ctx.error_flags() == 0
    # under capture a malformed tree runs as a chain and a bad path leaves the request untouched: both raise bit 3
    par_s.copy_(torch.tensor([[-1] + list(range(T - 1)), [0] * T], dtype=torch.int32))
    nodes_s.zero_(), cnt_s.copy_(torch.tensor([1, T + 1], dtype=torch.int32))
    gT.replay()
    assert ctx.error_flags() & 8


def test_tree_steps_then_spill(cuda_lib):
    """Tree steps of 6 nodes with accepts until the window is full, then a spill: the spilled rows are the accepted keys and
    values, and the tables equal a rebuild over the stored keys."""
    B, Hq, Hkv, n, K, L, gen, T = 2, 8, 2, 1500, 8, 40, 24, 6
    r = Run(B, Hq, Hkv, n, K, L, 2048, gen, seed=5)
    r.ctx.reserve_query_tokens(T)
    rng = random.Random(9)
    used = 0
    while used + T <= gen:
        pars = [random_tree(T, rng) for _ in range(B)]
        depth = min(len(root_path(p, T - 1)) for p in pars)
        paths = [root_path(p, T - 1)[:depth] for p in pars]   # the same count for every request
        q = torch.randn((B, T, Hq, d), generator=r.g).bfloat16()
        k = torch.randn((B, T, Hkv, d), generator=r.g).bfloat16()
        v = torch.randn((B, T, Hkv, d), generator=r.g).bfloat16()
        r.ctx.plan(T, parents=torch.tensor(pars, dtype=torch.int32, device=DEV))
        r.ctx.decode_tokens(1, T, q.to(DEV), k.to(DEV), v.to(DEV))
        nodes = torch.tensor([p + [0] * (T - len(p)) for p in paths], dtype=torch.int32, device=DEV)
        r.ctx.accept(nodes, torch.full((B,), depth, dtype=torch.int32, device=DEV))
        for i in range(depth):
            idx = torch.tensor([p[i] for p in paths])
            r.push(torch.stack([k[b, idx[b]] for b in range(B)])[:, :, None], torch.stack([v[b, idx[b]] for b in range(B)])[:, :, None])
        used += depth
    n_old = r.n_off
    g, (rk, rv) = r.spill()
    assert g == used
    k_st, v_st, _ = (x.cpu() for x in r.ctx.read_cache(1))
    assert torch.equal(k_st[:, :, n_old:n_old + g], rk)
    assert torch.equal(v_st[:, :, n_old:n_old + g], rv)
    assert_tables_equal(lsh_tables(r.ctx, 1), lsh_tables(r.rebuild(), 1), range(B))
    assert r.ctx.error_flags() == 0


def test_tree_refusals(cuda_lib):
    """Malformed trees and paths leave the state unchanged (a twin that never saw them then matches bitwise), raise bit 3 and
    MPIG_EINVAL; rewind after plan_tree, a second accept and T above the reserve are refused."""
    B, Hq, Hkv, T = 2, 8, 2, 4
    tw = twins(B, Hq, Hkv, 1500, 8, 40, T, seed=9)
    ctx, twin = tw.tok, tw.seq
    q, k, v = tw.inputs(T)
    qd, kd, vd = q.to(DEV), k.to(DEV), v.to(DEV)
    for bad in ([[-1, 0, 1, 2], [0, 0, 1, 2]], [[-1, 0, 2, 1], [-1, 0, 0, 0]], [[-1, 0, 1, 2], [-1, 0, 1, -1]]):
        with pytest.raises(N.MagicPigError, match="malformed"):
            ctx.plan(T, parents=torch.tensor(bad, dtype=torch.int32, device=DEV))
    assert ctx.error_flags() & 8
    with pytest.raises(N.MagicPigError, match="outside"):
        ctx.plan(T + 1, parents=torch.full((B, T + 1), -1, dtype=torch.int32, device=DEV))
    pars = [[-1, 0, 0, 1], [-1, 0, 1, 1]]
    for c in (ctx, twin):
        c.plan(T, parents=torch.tensor(pars, dtype=torch.int32, device=DEV))
        c.decode_tokens(1, T, qd, kd, vd)
        c.dense_decode_tokens(0, T, qd, kd, vd)
    with pytest.raises(N.MagicPigError, match="is a tree"):
        ctx.rewind(torch.zeros(B, dtype=torch.int32, device=DEV))
    # request 0: 0 -> {1, 2}, 1 -> {3}; request 1: 0 -> {1}, 1 -> {2, 3}
    good = torch.tensor([[0, 1, 3, 0], [0, 1, 2, 0]], dtype=torch.int32, device=DEV)
    for nodes, cnt in (([[0, 2, 1, 0], [0, 1, 2, 0]], [3, 3]),    # 1 is not a child of 2
                       ([[0, 1, 3, 0], [1, 2, 0, 0]], [3, 2]),    # a path that does not start at the root
                       ([[0, 1, 3, 0], [0, 1, 2, 0]], [3, 5]),    # count above T
                       ([[0, 3, 0, 0], [0, 1, 2, 0]], [2, 3])):   # 3's parent is 1, not 0
        with pytest.raises(N.MagicPigError, match="root path"):
            ctx.accept(torch.tensor(nodes, dtype=torch.int32, device=DEV), torch.tensor(cnt, dtype=torch.int32, device=DEV))
    cnt = torch.tensor([3, 3], dtype=torch.int32, device=DEV)
    ctx.accept(good, cnt)                                             # the refused accept may be repeated
    twin.accept(good, cnt)
    with pytest.raises(N.MagicPigError, match="at most one rewind or accept"):
        ctx.accept(good, cnt)
    next_steps_equal(ctx, twin, B, Hq, Hkv, torch.Generator().manual_seed(3))
    assert twin.error_flags() == 0
    # clear() forgets a pending tree: rewind is accepted again after a chain plan
    ctx.plan(T, parents=torch.tensor(pars, dtype=torch.int32, device=DEV))
    ctx.clear()
    ctx.plan(2)
    ctx.rewind(torch.zeros(B, dtype=torch.int32, device=DEV))


def test_dropin_tree_loop(cuda_lib):
    """LSHSparseAttnServer(max_query_tokens=6) on a 3-layer config with generation_buffer = 16: a scripted tree loop across spills.
    Every accepted node's output is within one bf16 ulp of a twin server that generates the path one token at a time."""
    from magicpig_b200.attnserver import LSHSparseAttnServer
    cfg = _Cfg()
    K, L, B, P, M, gen, T = 8, 40, 2, 600, 1024, 16, 6
    Hq, Hkv = cfg.num_attention_heads, cfg.num_key_value_heads
    hf = synth.make_hash_func(d, K, L, seed=41)
    g = torch.Generator().manual_seed(42)
    kc = [torch.randn((B, P, Hkv, d), generator=g).bfloat16() for _ in range(3)]
    vc = [torch.randn((B, P, Hkv, d), generator=g).bfloat16() for _ in range(3)]
    servers = []
    for mq in (T, 1):
        s = LSHSparseAttnServer(cfg, K=K, L=L, batch_size=B, generation_buffer=gen, max_length=M, dense_layers=(0,),
                                device=DEV, hash_func=hf.to(DEV), max_query_tokens=mq)
        s.alloc_buffer(P)
        for layer in range(3):
            for b in range(B):
                s.fill(layer, b, kc[layer][b].to(DEV), vc[layer][b].to(DEV), P)
                s.build_table(layer, b, P)
        servers.append(s)
    spec, twin = servers
    rng = random.Random(8)
    accepted_total, used = 0, 0
    for step in range(14):
        if used + T > gen:
            spec.spill_window()
            twin.spill_window()
            used = 0
        pars = random_tree(T, rng)                       # one (T,) tree for every request
        path = root_path(pars, rng.randrange(T))
        q = [torch.randn((B, Hq, T, d), generator=g).bfloat16().to(DEV) for _ in range(3)]
        k = [torch.randn((B, Hkv, T, d), generator=g).bfloat16().to(DEV) for _ in range(3)]
        v = [torch.randn((B, Hkv, T, d), generator=g).bfloat16().to(DEV) for _ in range(3)]
        spec.plan(T, parents=pars)
        outs = [spec.decode(q[l], k[l], v[l], l).clone() for l in range(3)]
        spec.accept(path, len(path))
        for t in path:
            twin.plan()
            for l in range(3):
                o = twin.decode(q[l][:, :, t:t + 1], k[l][:, :, t:t + 1], v[l][:, :, t:t + 1], l)
                a, b_ = outs[l][:, t].float(), o[:, 0].float()
                bound = torch.maximum(a.abs(), b_.abs()) * 2.0 ** -7 + 1e-5 * b_.abs().amax(dim=-1, keepdim=True)
                assert bool(((a - b_).abs() <= bound).all()), (step, l, t)
        used += len(path)
        accepted_total += len(path)
    assert accepted_total > gen


def test_runner_step_tree(cuda_lib):
    """step_tree on a chain equals step_tokens bitwise; on a branching tree each node's logits match step_tokens over its path
    within 2e-2, and after accepting a path the next step matches a twin that ran the path as a chain."""
    from magicpig_b200.llama_runner import LlamaDecodeRunner, LlamaShape
    shape = LlamaShape("tiny", 2, 512, 1024, 4, 2, 1000, 500000.0, 1e-5)
    B, P, T = 2, 300, 5
    runners = [LlamaDecodeRunner(shape, 6, 16, B, 1024, seed=3, generation_buffer=64, dense_layers=(0,), fused=False,
                                 max_query_tokens=T) for _ in range(2)]
    for r in runners:
        r.synthetic_prefill(P, seed=9)
    spec, twin = runners
    gen = torch.Generator().manual_seed(4)
    ids = torch.randint(0, shape.vocab_size, (B, T), generator=gen).to(DEV)
    full = torch.full((B,), T, dtype=torch.int32, device=DEV)
    spec.ids_tok[:, :T].copy_(ids)
    twin.ids_tok[:, :T].copy_(ids)
    chain = torch.tensor([-1] + list(range(T - 1)), dtype=torch.int32, device=DEV)
    a = spec.step_tree(T, chain, torch.zeros((B, T), dtype=torch.int32, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV)).clone()
    b_ = twin.step_tokens(T, drop=full).clone()
    assert torch.equal(a, b_)
    assert torch.equal(spec.pos.cpu(), twin.pos.cpu())
    pars = [-1, 0, 0, 1, 2]
    got = spec.step_tree(T, pars).clone()   # no accept: every node stays until the accept below
    for t in range(T):
        path = root_path(pars, t)
        twin.ids_tok[:, :len(path)].copy_(ids[:, path])
        ref = twin.step_tokens(len(path), drop=torch.full((B,), len(path), dtype=torch.int32, device=DEV))
        assert rel_max(got[:, t], ref[:, len(path) - 1]) <= 2e-2, t
    path = root_path(pars, 4)
    spec.server.accept(path, len(path))
    spec.pos.sub_(T - len(path))
    twin.ids_tok[:, :len(path)].copy_(ids[:, path])
    twin.step_tokens(len(path), drop=torch.zeros(B, dtype=torch.int32, device=DEV))
    assert torch.equal(spec.pos.cpu(), twin.pos.cpu())
    nxt = torch.randint(0, shape.vocab_size, (B, 1), generator=gen).to(DEV)
    spec.ids_tok[:, :1].copy_(nxt)
    twin.ids_tok[:, :1].copy_(nxt)
    assert rel_max(spec.step_tokens(1).clone(), twin.step_tokens(1).clone()) <= 2e-2
