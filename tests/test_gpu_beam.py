"""Device-side reorder of a batch's requests (`-m gpu`): mpig_reorder_requests against a twin that applies the same map with one
mpig_fork_request per moved request.

A reorder is exactly the forks it stands for, so every later output of the context is compared BITWISE with the twin's: codes, nnz,
index lists, fp32 and bf16 outputs of the sparse layer and fp32 and bf16 outputs of the dense layer, over single-token steps,
T-token steps with rewind and token trees with accept, across reorders by random valid maps, including moves across context slots.
Covered: fused_kreg 0 / 1, a full dense cache per request (R = 0), the shared dense mode (R > 0), shared spill with private keys
spilled before and after the reorders, the three-launch path; one moved request against the oracle; a captured plan -> layers ->
reorder replayed with different maps; the refusals; the host mirrors after a captured reorder; and a width-4 beam search of the
Llama runner (one captured step() + beam_step) against a runner that forks on the host.
"""
import random

import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200.ops import Context
from tests.support.fp64 import assert_1e3_f32, oracle_decode
from tests.support.library import DEV, NL, NS, Doc, d, two_layer_context

pytestmark = pytest.mark.gpu
GEN = 64
Hq, Hkv, K, L, M, N_KEYS, P_DENSE = 8, 2, 8, 60, 4096, 2000, 300
B, C = 4, 2


def make_ctx(hf, C=C, R=0, spill=False, impl=1, kreg=0):
    return two_layer_context(K, L, Hq, Hkv, B, M, GEN, hf, dict(decode_impl=impl, fused_kreg=kreg, out_f32=1, save_mask=1),
                             alloc_dense_kv=True, max_query_tokens=4, num_contexts=C, dense_tail_rows=R, shared_spill=spill)


def fill(ctx, docs, wins):
    """slot c holds docs[c] (filled through request c); request b gets its own window wins[b] and the dense prefix of its slot's
    document (the initial binding is b mod C)"""
    for c, doc in enumerate(docs):
        doc.fill_store(ctx, c)
    for b in range(B):
        doc = docs[b % C]
        ctx.window_fill(1, b, doc.avg.to(DEV).contiguous(), wins[b][0].to(DEV).contiguous(), wins[b][1].to(DEV).contiguous())
        ctx.dense_fill(0, b, doc.dk.to(DEV), doc.dv.to(DEV), P_DENSE)


def random_map(rng, n=B):
    """a random map obeying the rule: a non-empty set of fixed points, every other request copies one of them"""
    fixed = rng.sample(range(n), rng.randint(1, n))
    return [b if b in fixed else rng.choice(fixed) for b in range(n)]


class Pair:
    """A context that reorders and its twin that forks, driven with the same inputs; every output is compared bitwise."""

    def __init__(self, ctx, twin, seed):
        self.a, self.t = ctx, twin
        self.g = torch.Generator().manual_seed(seed)
        self.rng = random.Random(seed)

    def qkv(self, T=1):
        q = torch.randn((B, T, Hq, d), generator=self.g).bfloat16().to(DEV)
        k = torch.randn((B, T, Hkv, d), generator=self.g).bfloat16().to(DEV)
        v = torch.randn((B, T, Hkv, d), generator=self.g).bfloat16().to(DEV)
        return q, k, v

    def reorder(self, src_of):
        self.a.reorder(torch.tensor(src_of, dtype=torch.int32, device=DEV))
        for b, s in enumerate(src_of):
            if s != b:
                self.t.fork(s, b)

    def run(self, T=1, parents=None):
        """one step of T tokens (tree when parents is given) on both contexts; returns nothing, asserts equality"""
        q, k, v = self.qkv(T)
        outs = []
        for ctx in (self.a, self.t):
            if parents is not None:
                ctx.plan(T, parents=parents)
            else:
                ctx.plan(T)
            if T == 1:
                od = ctx.dense_decode(0, q[:, 0], k[:, 0], v[:, 0])
                fd = ctx.last_out_f32()
                os_ = ctx.decode(1, q[:, 0], k[:, 0], v[:, 0])
            else:
                od = ctx.dense_decode_tokens(0, T, q, k, v)
                fd = ctx.last_out_f32()
                os_ = ctx.decode_tokens(1, T, q, k, v)
            nz, res = ctx.last_probe(True)
            outs.append(dict(od=od.clone(), fd=fd, os=os_.clone(), fs=ctx.last_out_f32(), nz=nz, res=res,
                             codes=ctx.last_codes() if ctx.get_info("last_decode_fused") else None))
        x, y = outs
        assert torch.equal(x["nz"], y["nz"]), "nnz differ"
        valid = torch.arange(M, device=DEV)[None] < x["nz"][:, None]
        assert torch.equal(torch.where(valid, x["res"], -1), torch.where(valid, y["res"], -1)), "index lists differ"
        if x["codes"] is not None:
            assert torch.equal(x["codes"], y["codes"]), "codes differ"
        for key in ("od", "fd", "os", "fs"):
            assert torch.equal(x[key], y[key]), f"{key} differs"

    def single(self):
        self.run(1)

    def tokens(self):
        self.run(4)
        drop = torch.tensor([self.rng.randint(0, 4) for _ in range(B)], dtype=torch.int32, device=DEV)
        for ctx in (self.a, self.t):
            ctx.rewind(drop)

    def tree(self):
        par = torch.tensor([[-1, 0, 0, 1]] * B, dtype=torch.int32, device=DEV)
        self.run(4, parents=par)
        paths = [[0], [0, 1], [0, 2], [0, 1, 3]]
        pick = [paths[self.rng.randrange(4)] for _ in range(B)]
        nodes = torch.tensor([p + [0] * (4 - len(p)) for p in pick], dtype=torch.int32, device=DEV)
        count = torch.tensor([len(p) for p in pick], dtype=torch.int32, device=DEV)
        for ctx in (self.a, self.t):
            ctx.accept(nodes, count)

    def spill(self):
        assert self.a.spill_window().tolist() == self.t.spill_window().tolist()


def setup(hf, seed, **kw):
    docs = [Doc(Hkv, N_KEYS, K, L, hf, seed + 10 * c, P_dense=P_DENSE) for c in range(C)]
    g = torch.Generator().manual_seed(seed + 99)
    wins = [(torch.randn((Hkv, NS + NL, d), generator=g).bfloat16(), torch.randn((Hkv, NS + NL, d), generator=g).bfloat16())
            for _ in range(B)]
    ctx, twin = make_ctx(hf, **kw), make_ctx(hf, **kw)
    for c in (ctx, twin):
        fill(c, docs, wins)
    return ctx, twin, docs, wins


VARIANTS = {
    "full_dense": dict(),
    "kreg": dict(kreg=1),
    "dense_tail": dict(R=96),
    "shared_spill": dict(spill=True),
    "three_launch": dict(impl=0),
}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_reorder_equals_forks(cuda_lib, variant):
    kw = VARIANTS[variant]
    hf = torch.randn((d, K * L), generator=torch.Generator().manual_seed(1)).bfloat16()
    ctx, twin, _, _ = setup(hf, 5, **kw)
    p = Pair(ctx, twin, 7)
    multi = kw.get("impl", 1) == 1   # T-token steps need the fused kernel
    spill = kw.get("spill", False)
    cross = [0, 0, 2, 2]   # requests 1 and 3 (slot 1) move to slot 0
    assert [b % C for b in range(B)] == [0, 1, 0, 1]
    for rnd in range(3):
        p.single()
        if spill:
            p.spill()      # private keys spilled before the reorder
        p.reorder(cross if rnd == 0 else random_map(p.rng))
        p.single()
        if multi:
            p.tokens()
            p.tree()
        p.reorder(random_map(p.rng))
        if spill:
            p.single()
            p.spill()      # ... and after it
        p.single()
        if multi:
            p.tree()
            p.tokens()
        p.single()
    for c in (ctx, twin):
        assert c.error_flags() == 0
    p.reorder([1, 1, 1, 1])   # every request takes request 1's sequence (slot 1)
    p.single()


def test_oracle_moved_request(cuda_lib):
    """A request moved across slots decodes over its new slot's store and its source's window: within 1e-3 of the oracle fed
    the twin's stored state and host copies of the windows."""
    hf = torch.randn((d, K * L), generator=torch.Generator().manual_seed(3)).bfloat16()
    ctx, twin, docs, wins = setup(hf, 21)
    p = Pair(ctx, twin, 4)
    g = torch.Generator().manual_seed(6)
    win = [(wk.clone(), wv.clone()) for wk, wv in wins]
    slot = [b % C for b in range(B)]

    def step(check=()):
        q, k, v = (x.to(DEV) for x in (torch.randn((B, Hq, d), generator=g).bfloat16(), torch.randn((B, Hkv, d), generator=g).bfloat16(),
                                       torch.randn((B, Hkv, d), generator=g).bfloat16()))
        for c in (ctx, twin):
            c.plan()
            c.dense_decode(0, q, k, v)
            c.decode(1, q, k, v)
        assert torch.equal(ctx.last_out_f32(), twin.last_out_f32())
        k_st, v_st, kn_st = (x.cpu() for x in twin.read_cache(1))
        for b in range(B):
            doc = docs[slot[b]]
            avg = doc.avg.reshape(1, Hkv, 1, d)
            kb, vb, qb = k[b].cpu().reshape(1, Hkv, 1, d), v[b].cpu().reshape(1, Hkv, 1, d), q[b].cpu().reshape(1, Hq, 1, d)
            if b in check:
                n = doc.n
                kd = k_st[slot[b], :, :n].contiguous()
                t = dict(B=1, Hq=Hq, Hkv=Hkv, d=d, K=K, L=L, n=n, M=M, hash_func=hf, kcodes=doc.kcodes[None], key=kd[None],
                         value=v_st[slot[b], :, :n][None].contiguous(), key_norm=kn_st[slot[b], :, :n][None].contiguous(), avg_k=avg)
                _, nz_ref, _, o_exact = oracle_decode(t, qb, kb, vb, win[b][0][None], win[b][1][None], Hq // Hkv)
                rows = slice(b * Hq, (b + 1) * Hq)
                assert torch.equal(ctx.last_probe()[0].cpu()[rows], nz_ref)
                assert_1e3_f32(ctx.last_out_f32()[rows].cpu(), o_exact)
            win[b] = (torch.cat([win[b][0], (kb - avg)[0]], dim=1), torch.cat([win[b][1], vb[0]], dim=1))

    step()
    step()
    p.reorder([0, 1, 2, 0])   # request 3 leaves slot 1 for request 0's sequence on slot 0
    win[3], slot[3] = (win[0][0].clone(), win[0][1].clone()), slot[0]
    step(check=(3,))
    step(check=(0, 3))


def test_graph_replays_with_new_maps(cuda_lib):
    """plan -> dense and sparse layer -> reorder, captured once (R > 0 and shared spill), replayed with different map contents:
    every replay equals the eager twin's plan, layers and forks."""
    hf = torch.randn((d, K * L), generator=torch.Generator().manual_seed(9)).bfloat16()
    ctx, twin, _, _ = setup(hf, 31, R=96, spill=True)
    Pair(ctx, twin, 30).single()   # every kernel has run once before the capture
    g = torch.Generator().manual_seed(10)
    q = torch.zeros((B, Hq, d), dtype=torch.bfloat16, device=DEV)
    k = torch.zeros((B, Hkv, d), dtype=torch.bfloat16, device=DEV)
    v = torch.zeros((B, Hkv, d), dtype=torch.bfloat16, device=DEV)
    src = torch.arange(B, dtype=torch.int32, device=DEV)
    od = torch.empty((B, Hq * d), dtype=torch.bfloat16, device=DEV)
    os_ = torch.empty((B, Hq * d), dtype=torch.bfloat16, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            ctx.plan()
            ctx.dense_decode(0, q, k, v, od)
            ctx.decode(1, q, k, v, os_)
            ctx.reorder(src)
    torch.cuda.synchronize()
    rng = random.Random(11)
    for step in range(12):
        for x in (q, k, v):
            x.copy_(torch.randn(x.shape, generator=g).bfloat16())
        m = random_map(rng) if step % 3 else list(range(B))
        src.copy_(torch.tensor(m, dtype=torch.int32))
        graph.replay()
        twin.plan()
        td = twin.dense_decode(0, q, k, v).clone()
        ts = twin.decode(1, q, k, v).clone()
        nz_t = twin.last_probe()[0]
        for b, sb in enumerate(m):
            if sb != b:
                twin.fork(sb, b)
        torch.cuda.synchronize()
        assert torch.equal(od, td) and torch.equal(os_, ts), f"step {step}"
        assert torch.equal(ctx.last_probe()[0], nz_t)
        if step == 5:
            assert ctx.spill_window().tolist() == twin.spill_window().tolist()   # reads the device lengths and maps
    assert ctx.error_flags() == 0 and twin.error_flags() == 0


def state_equal(ctx, twin, seed):
    """one more single-token step, compared bitwise"""
    Pair(ctx, twin, seed).single()


def test_refusals(cuda_lib):
    hf = torch.randn((d, K * L), generator=torch.Generator().manual_seed(12)).bfloat16()
    ctx, twin, _, _ = setup(hf, 41, R=96, spill=True)
    p = Pair(ctx, twin, 13)
    p.single()
    for bad in ([0, 4, 2, 3], [-1, 1, 2, 3], [1, 2, 2, 3]):   # out of range (both ways); a source (1) that is itself moved
        with pytest.raises(N.MagicPigError, match="code -1"):
            ctx.reorder(torch.tensor(bad, dtype=torch.int32, device=DEV))
        assert ctx.error_flags() & 16
        state_equal(ctx, twin, 14)
    # under capture the kernel's own check leaves every request untouched
    bad = torch.tensor([1, 2, 2, 3], dtype=torch.int32, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            ctx.reorder(bad)
    torch.cuda.synchronize()
    ctx.clear()
    twin.clear()
    docs = [Doc(Hkv, N_KEYS, K, L, hf, 41 + 10 * c, P_dense=P_DENSE) for c in range(C)]
    g = torch.Generator().manual_seed(41 + 99)
    wins = [(torch.randn((Hkv, NS + NL, d), generator=g).bfloat16(), torch.randn((Hkv, NS + NL, d), generator=g).bfloat16())
            for _ in range(B)]
    for c in (ctx, twin):
        fill(c, docs, wins)
    graph.replay()
    assert ctx.error_flags() & 16
    state_equal(ctx, twin, 15)
    p.single()
    bad.copy_(torch.tensor([0, 0, 2, 2], dtype=torch.int32))   # now valid: the same graph applies it
    graph.replay()
    p.t.fork(0, 1)
    p.t.fork(2, 3)
    state_equal(ctx, twin, 16)
    # fixed bindings
    own = Context(K, L, 2, Hq, Hkv, d, B, M, NS, NL, GEN, dense_layers=[0], alloc_dense_kv=True, device=DEV)
    with pytest.raises(N.MagicPigError, match="code -4"):
        own.reorder(torch.arange(B, dtype=torch.int32, device=DEV))
    # the reorder ends the pending step
    q, k, v = p.qkv(4)
    ctx.plan(4)
    ctx.dense_decode_tokens(0, 4, q, k, v)
    ctx.decode_tokens(1, 4, q, k, v)
    ctx.reorder(torch.arange(B, dtype=torch.int32, device=DEV))
    with pytest.raises(N.MagicPigError, match="code -4"):
        ctx.rewind(torch.zeros(B, dtype=torch.int32, device=DEV))
    nodes = torch.zeros((B, 4), dtype=torch.int32, device=DEV)
    with pytest.raises(N.MagicPigError, match="code -4"):
        N.check(ctx.lib.mpig_accept(ctx._h, nodes.data_ptr(), torch.ones(B, dtype=torch.int32, device=DEV).data_ptr(), None), "mpig_accept")
    with pytest.raises(N.MagicPigError, match="code -1"):
        N.check(ctx.lib.mpig_reorder_requests(ctx._h, None, None), "mpig_reorder_requests")


def test_host_mirrors_after_captured_reorder(cuda_lib):
    """A captured reorder moves request 3 from slot 1 to slot 0 on the device only; a fill through request 3 must then write
    slot 0, and a spill must stage its keys there (shared spill mode, shared dense mode)."""
    hf = torch.randn((d, K * L), generator=torch.Generator().manual_seed(17)).bfloat16()
    ctx, twin, docs, _ = setup(hf, 51, R=96, spill=True)
    p = Pair(ctx, twin, 18)
    p.single()
    src = torch.tensor([0, 1, 2, 0], dtype=torch.int32, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            ctx.reorder(src)
    torch.cuda.synchronize()
    graph.replay()
    twin.fork(0, 3)
    p.single()
    new = Doc(Hkv, N_KEYS, K, L, hf, 77, P_dense=P_DENSE)
    for c in (ctx, twin):
        new.fill_store(c, 3)                                   # slot 0 (request 3's binding after the reorder)
        c.dense_fill(0, 3, new.dk.to(DEV), new.dv.to(DEV), P_DENSE)
    for c in (ctx, twin):
        k_, v_, kn_ = c.read_cache(1)
        assert torch.equal(k_[0, :, :N_KEYS].cpu(), new.key) and torch.equal(k_[1, :, :N_KEYS].cpu(), docs[1].key)
    for _ in range(4):
        p.single()
    p.spill()
    for x, y in zip(ctx.read_cache(1), twin.read_cache(1)):
        assert torch.equal(x, y)
    for _ in range(3):
        p.single()
    assert ctx.error_flags() == 0


def test_runner_beam_search(cuda_lib):
    """A width-4 beam search over a small random-weight model in shared spill mode: 64 replays of one captured step() +
    beam_step, with spills between them, against a runner that replays a captured step() alone, reads the parents to the host and
    forks.  Tokens, scores and logits are bitwise equal."""
    from magicpig_b200.attnserver import beam_sources
    from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner
    W, P, gen_buf = 4, 3000, 16
    runs = [LlamaDecodeRunner(LLAMA31_8B, 8, 60, W, 4096, device=DEV, num_layers=3, num_contexts=1, generation_buffer=gen_buf,
                              shared_spill=True, dense_tail_rows=128) for _ in range(2)]
    scores = [torch.zeros(W, dtype=torch.float32, device=DEV) for _ in range(2)]
    runs[0].synthetic_prefill(P, shared=True)
    runs[0].capture(beam_scores=scores[0])
    runs[1].synthetic_prefill(P, shared=True)
    runs[1].capture()
    for r, sc in zip(runs, scores):   # the warm-up steps moved the beams: start again from the prompt
        r.server.clear()
        r.synthetic_prefill(P, shared=True)
        r.ids.fill_(17)
        sc.copy_(torch.tensor([0.0] + [float("-inf")] * (W - 1)))
    a, b = runs
    for step in range(64):
        if step % 10 == 9:
            assert a.server.spill_window().tolist() == b.server.spill_window().tolist()
        a.replay()
        b.replay()
        parents, tokens, new = b.beam_select(scores[1])
        src_of, request_of = beam_sources(parents)
        for dst, s_ in enumerate(src_of.tolist()):
            if s_ != dst:
                b.fork(s_, dst)
        b.ids[request_of.long(), 0] = tokens
        scores[1][request_of.long()] = new
        torch.cuda.synchronize()
        assert torch.equal(a.logits, b.logits), f"step {step}: logits"
        assert torch.equal(a.ids, b.ids), f"step {step}: tokens"
        assert torch.equal(scores[0], scores[1]), f"step {step}: scores"
        assert torch.equal(a.pos, b.pos)
    assert bool(torch.isfinite(scores[0]).all())
    for r in runs:
        assert r.server.ctx.error_flags() == 0
