"""Shared dense prefix (`-m gpu`): with dense_tail_rows R > 0 the dense layers keep a slot's prompt rows once, and every request
only the rows it adds after its prompt.

Every check compares a shared-dense context (C < B slots, filled through a few requests, then fork / bind) against a twin that holds
one slot and one full dense cache per request (R = 0, every request filled), given the same q / k / v.  The shared-dense kernel
sums in another order, so dense fp32 outputs agree within 1e-5 (absolute); sparse layers in the same context stay bitwise equal.
Dense outputs also agree within 1e-3 with an fp64 torch restatement over each request's full rows.
"""
import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200 import synth
from magicpig_b200.ops import Context
from tests.support.library import DEV, NL, NS, Doc, _Cfg, assert_lists_equal, d, two_layer_context

pytestmark = pytest.mark.gpu
GEN = 32
TOL = 1e-5


def make_ctx(B, C, Hq, Hkv, M, K, L, hf, R=0, t_max=1, gen=GEN):
    return two_layer_context(K, L, Hq, Hkv, B, M, gen, hf, dict(out_f32=1, save_mask=1), alloc_dense_kv=True,
                             max_query_tokens=t_max, num_contexts=C, dense_tail_rows=R)


def dense_ref(q, rows_k, rows_v, G):
    """fp64 softmax attention of q (Hq, d) over rows (n, Hkv, d)."""
    k = rows_k.double().repeat_interleave(G, dim=1)   # (n, Hq, d)
    v = rows_v.double().repeat_interleave(G, dim=1)
    s = torch.einsum("hd,nhd->hn", q.double(), k) / d ** 0.5
    return torch.einsum("hn,nhd->hd", torch.softmax(s, dim=-1), v)


class DensePair:
    """A shared-dense context and its twin.  docs_of[b] = the document of request b; the shared context is filled through the
    requests in `fill` and forked along `forks`; the twin fills every request.  rows[b] mirrors request b's dense rows on the host
    (for single-token steps) for the fp64 restatement."""

    def __init__(self, B, C, Hq, Hkv, docs_of, forks, fill, R=GEN + 8, t_max=1, n=1500, K=8, L=60, seed=0, binds=(), P=300):
        self.B, self.Hq, self.Hkv, self.G = B, Hq, Hkv, Hq // Hkv
        self.hf = synth.make_hash_func(d, K, L, seed=seed + 11)
        M = n + 256
        self.docs = {i: Doc(Hkv, n, K, L, self.hf, seed + 100 * (i + 1), P_dense=P) for i in set(docs_of)}
        self.sh = make_ctx(B, C, Hq, Hkv, M, K, L, self.hf, R, t_max)
        self.tw = make_ctx(B, 0, Hq, Hkv, M, K, L, self.hf, 0, t_max)
        for b, slot in binds:
            self.sh.bind(b, slot)
        for b in fill:
            self.docs[docs_of[b]].fill_store(self.sh, b)
            self.docs[docs_of[b]].fill_request(self.sh, b)
        for src, dst in forks:
            self.sh.fork(src, dst)
        for b in range(B):
            self.docs[docs_of[b]].fill_store(self.tw, b)
            self.docs[docs_of[b]].fill_request(self.tw, b)
        self.rows = [[self.docs[docs_of[b]].dk.clone(), self.docs[docs_of[b]].dv.clone()] for b in range(B)]
        self.g = torch.Generator().manual_seed(seed + 7)

    def qkv(self, T=1):
        B, Hq, Hkv, g = self.B, self.Hq, self.Hkv, self.g
        return (torch.randn((B, T, Hq, d), generator=g).bfloat16().to(DEV), torch.randn((B, T, Hkv, d), generator=g).bfloat16().to(DEV),
                torch.randn((B, T, Hkv, d), generator=g).bfloat16().to(DEV))

    def compare_dense(self):
        a, b = self.sh.last_out_f32(), self.tw.last_out_f32()
        assert torch.isfinite(a).all()
        assert torch.allclose(a, b, rtol=0, atol=TOL), f"dense fp32 outputs differ by {(a - b).abs().max().item()}"
        return a

    def single(self, sparse=True, ref=True):
        if sparse:
            q, k, v = self.qkv()
            outs = []
            for ctx in (self.sh, self.tw):
                ctx.plan()
                outs.append(ctx.decode(1, q[:, 0], k[:, 0], v[:, 0]).clone())
            assert_lists_equal(*self.sh.last_probe(True), *self.tw.last_probe(True))
            assert torch.equal(self.sh.last_out_f32(), self.tw.last_out_f32())
            assert torch.equal(outs[0], outs[1])
        else:
            for ctx in (self.sh, self.tw):
                ctx.plan()
        q, k, v = self.qkv()
        for ctx in (self.sh, self.tw):
            ctx.dense_decode(0, q[:, 0], k[:, 0], v[:, 0])
        out = self.compare_dense().reshape(self.B, self.Hq, d)
        for b in range(self.B):
            self.rows[b][0] = torch.cat([self.rows[b][0], k[b, 0][None].cpu()])
            self.rows[b][1] = torch.cat([self.rows[b][1], v[b, 0][None].cpu()])
            if ref:
                r = dense_ref(q[b, 0].cpu(), *self.rows[b], self.G)
                assert (out[b].cpu().double() - r).abs().max().item() < 1e-3

    def tokens(self, T, drop):
        q, k, v = self.qkv(T)
        for ctx in (self.sh, self.tw):
            ctx.plan(T)
            ctx.dense_decode_tokens(0, T, q, k, v)
        self.compare_dense()
        dr = torch.tensor(drop, dtype=torch.int32, device=DEV)
        for ctx in (self.sh, self.tw):
            ctx.rewind(dr)

    def tree(self, parents, nodes, count):
        T = len(parents)
        par = torch.tensor([parents] * self.B, dtype=torch.int32, device=DEV)
        q, k, v = self.qkv(T)
        for ctx in (self.sh, self.tw):
            ctx.plan(T, parents=par)
            ctx.dense_decode_tokens(0, T, q, k, v)
        self.compare_dense()
        nd = torch.tensor([nodes + [0] * (T - len(nodes))] * self.B, dtype=torch.int32, device=DEV)
        ct = torch.tensor(count, dtype=torch.int32, device=DEV)
        for ctx in (self.sh, self.tw):
            ctx.accept(nd, ct)


@pytest.mark.parametrize("G", [4, 8])
@pytest.mark.parametrize("B,C", [(4, 1), (8, 2)])
def test_fork_twin_single(cuda_lib, B, C, G):
    Hkv = 2
    docs_of = [b % C for b in range(B)]
    forks = [(b % C, b) for b in range(C, B)]
    p = DensePair(B, C, G * Hkv, Hkv, docs_of, forks, fill=range(C))
    assert p.sh.dense_tail_rows == GEN + 8 and p.tw.dense_tail_rows == 0
    for _ in range(4):
        p.single()


@pytest.mark.parametrize("G,T", [(4, 2), (4, 4), (4, 8), (8, 4)])
def test_tokens_and_trees(cuda_lib, G, T):
    """T*G = 8, 16, 32: chunks of 4, 2 and 1 requests at G = 4, and of 1 at G = 8."""
    B, Hkv = 4, 2
    p = DensePair(B, 1, G * Hkv, Hkv, [0] * B, [(0, b) for b in range(1, B)], fill=[0], t_max=T, R=GEN + 2 * T + 8)
    gen = torch.Generator().manual_seed(T)
    p.tokens(T, torch.randint(0, T + 1, (B,), generator=gen).tolist())
    p.single(sparse=False, ref=False)
    parents = [-1] + [int(torch.randint(0, t, (1,), generator=gen)) for t in range(1, T)]
    path = [0]
    for t in range(1, T):
        if parents[t] == path[-1]:
            path.append(t)
    counts = [len(path), 1, max(len(path) - 1, 0), len(path)]
    p.tree(parents, path, counts)
    p.single(sparse=False, ref=False)   # the accepted and rewound tails are right
    p.tokens(T, [0] * B)
    p.single(sparse=False, ref=False)


def test_two_chunks(cuda_lib):
    """B = 12 on one slot at G = 4: two chunks (8 and 4 requests) of single-token steps."""
    B, Hkv = 12, 2
    p = DensePair(B, 1, 8, Hkv, [0] * B, [(0, b) for b in range(1, B)], fill=[0])
    for _ in range(3):
        p.single(sparse=False)


def test_mixed_bases(cuda_lib):
    """A refill of the slot through request 2 with a shorter prompt, then a fork from it: requests 0 / 1 keep their longer base
    over the slot's new rows, requests 2 / 3 have the shorter one."""
    B, Hkv, Hq, P, P2 = 4, 2, 8, 300, 200
    p = DensePair(B, 1, Hq, Hkv, [0] * B, [(0, 1)], fill=[0], P=P)
    g = torch.Generator().manual_seed(5)
    k2, v2 = torch.randn((P2, Hkv, d), generator=g).bfloat16(), torch.randn((P2, Hkv, d), generator=g).bfloat16()
    p.sh.dense_fill(0, 2, k2.to(DEV), v2.to(DEV), P2)
    p.sh.fork(2, 3)
    doc = p.docs[0]
    mixed_k, mixed_v = torch.cat([k2, doc.dk[P2:]]), torch.cat([v2, doc.dv[P2:]])
    for b in (0, 1):
        p.tw.dense_fill(0, b, mixed_k.to(DEV), mixed_v.to(DEV), P)
        p.rows[b] = [mixed_k.clone(), mixed_v.clone()]
    for b in (2, 3):
        p.tw.dense_fill(0, b, k2.to(DEV), v2.to(DEV), P2)
        p.rows[b] = [k2.clone(), v2.clone()]
    for _ in range(3):
        p.single(sparse=False)


def test_empty_member_and_other_slot(cuda_lib):
    """Request 3 has dense_len 0 at the decode (zeros); then it is bound to slot 1 and dense-filled there."""
    B, Hkv, Hq = 4, 2, 8
    p = DensePair(B, 2, Hq, Hkv, [0, 0, 0, 1], [(0, 1), (0, 2)], fill=[0], binds=[(3, 0)])
    for ctx in (p.sh, p.tw):
        ctx.dense_fill(0, 3, p.docs[1].dk.to(DEV), p.docs[1].dv.to(DEV), 0)
    for ctx in (p.sh, p.tw):
        ctx.plan()
        ctx.rewind(torch.tensor([0, 0, 0, 1], dtype=torch.int32, device=DEV))
    q, k, v = p.qkv()
    for ctx in (p.sh, p.tw):
        ctx.dense_decode(0, q[:, 0], k[:, 0], v[:, 0])
    out = p.compare_dense().reshape(B, Hq, d)
    assert torch.count_nonzero(out[3]) == 0 and torch.count_nonzero(out[0]) > 0
    # request 3 on its own slot, filled there
    p.sh.bind(3, 1)
    p.docs[1].fill_request(p.sh, 3)
    p.docs[1].fill_request(p.tw, 3)
    for b in range(3):
        p.rows[b] = None
    p.rows[3] = [p.docs[1].dk.clone(), p.docs[1].dv.clone()]
    for ctx in (p.sh, p.tw):
        ctx.plan()
    q, k, v = p.qkv()
    for ctx in (p.sh, p.tw):
        ctx.dense_decode(0, q[:, 0], k[:, 0], v[:, 0])
    out = p.compare_dense().reshape(B, Hq, d)
    rows_k = torch.cat([p.rows[3][0], k[3, 0][None].cpu()])
    rows_v = torch.cat([p.rows[3][1], v[3, 0][None].cpu()])
    assert (out[3].cpu().double() - dense_ref(q[3, 0].cpu(), rows_k, rows_v, 4)).abs().max().item() < 1e-3


def test_graph_replay_across_fork_and_bind(cuda_lib):
    """A dense step captured before a fork and a bind replays equal to an eager context after them."""
    B, Hkv, Hq, C = 4, 2, 8, 2
    hf = synth.make_hash_func(d, 8, 60, seed=3)
    docs = [Doc(Hkv, 1500, 8, 60, hf, 300 + i) for i in range(2)]
    ctxs = [make_ctx(B, C, Hq, Hkv, 1756, 8, 60, hf, R=40) for _ in range(2)]
    for c in ctxs:
        docs[0].fill_request(c, 0)
        docs[1].fill_request(c, 1)
        c.fork(0, 2)
        c.fork(1, 3)
    g = torch.Generator().manual_seed(9)
    q = torch.randn((B, Hq, d), generator=g).bfloat16().to(DEV)
    k = torch.randn((B, Hkv, d), generator=g).bfloat16().to(DEV)
    out = torch.empty((B, Hq * d), dtype=torch.bfloat16, device=DEV)
    cap, eager = ctxs
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):   # warm-up outside the capture (attribute setting), then one more step on the eager twin
        for c in ctxs:
            c.plan()
            c.dense_decode(0, q, k, k, out=out if c is cap else None)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap.plan()
        cap.dense_decode(0, q, k, k, out=out)
    for c in ctxs:
        c.fork(0, 3)   # request 3 moves to slot 0 with request 0's rows
        c.bind(2, 1)
        docs[1].fill_request(c, 2)
    for _ in range(3):
        graph.replay()
        eager.plan()
        ref = eager.dense_decode(0, q, k, k)
        torch.cuda.synchronize()
        assert torch.equal(out, ref)
        assert torch.equal(cap.last_out_f32(), eager.last_out_f32())


def test_capacity(cuda_lib):
    """The dense capacity of a request is base + R: an eager plan past it is refused with nothing changed; a captured plan
    saturates there, raises error flag bit 1, and every row access stays inside the tail."""
    B, Hkv, Hq, R = 4, 2, 8, 6
    p = DensePair(B, 1, Hq, Hkv, [0] * B, [(0, b) for b in range(1, B)], fill=[0], R=R)
    for _ in range(R):
        p.single(sparse=False, ref=False)
    with pytest.raises(N.MagicPigError, match="dense KV cache is full"):
        p.sh.plan()
    assert p.sh.error_flags() == 0
    # nothing changed: after a rewind of one token on both, the next step still matches the twin
    drop = torch.ones(B, dtype=torch.int32, device=DEV)
    for ctx in (p.sh, p.tw):
        ctx.rewind(drop)   # the refused plan left the last step pending
    for b in range(B):
        p.rows[b] = [r[:-1] for r in p.rows[b]]
    p.single(sparse=False)
    sh = p.sh
    g = torch.Generator().manual_seed(1)
    q = torch.randn((B, Hq, d), generator=g).bfloat16().to(DEV)
    k = torch.randn((B, Hkv, d), generator=g).bfloat16().to(DEV)
    out = torch.empty((B, Hq * d), dtype=torch.bfloat16, device=DEV)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sh.plan()
        sh.dense_decode(0, q, k, k, out=out)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert sh.error_flags() & 2
    o = sh.last_out_f32().reshape(B, Hq, d)
    assert torch.isfinite(o).all()
    # the saturated step overwrote the last tail row (R - 1) each time; the prompt rows are untouched: the output equals the
    # fp64 restatement over the prompt, the first R - 1 generated rows and the last k
    for b in range(B):
        rk = torch.cat([p.rows[b][0][:-1], k[b][None].cpu()])
        rv = torch.cat([p.rows[b][1][:-1], k[b][None].cpu()])
        assert (o[b].cpu().double() - dense_ref(q[b].cpu(), rk, rv, Hq // Hkv)).abs().max().item() < 1e-3


def test_exclusive_spill_until_dense_capacity(cuda_lib):
    """An exclusive request spills its sparse window and keeps decoding until its dense tail of R rows is used up."""
    K, L, n, Hq, Hkv, R = 8, 60, 1500, 8, 2, 40
    hf = synth.make_hash_func(d, K, L, seed=17)
    short = Doc(Hkv, n, K, L, hf, 500, w=NS + 8)
    long_ = Doc(Hkv, n, K, L, hf, 600, w=NS + NL + 6)
    sh = make_ctx(3, 2, Hq, Hkv, n + 256, K, L, hf, R=R)
    tw = make_ctx(3, 0, Hq, Hkv, n + 256, K, L, hf)
    sh.bind(1, 0)
    sh.bind(2, 1)            # request 2 alone on slot 1
    short.fill_store(sh, 0); short.fill_request(sh, 0); short.fill_request(sh, 1)
    long_.fill_store(sh, 2); long_.fill_request(sh, 2)
    for b, doc in ((0, short), (1, short), (2, long_)):
        doc.fill_store(tw, b); doc.fill_request(tw, b)
    gen = torch.Generator().manual_seed(3)
    steps = spilled = 0
    while True:
        if steps and steps % 20 == 0:
            a, b = sh.spill_window(), tw.spill_window()
            assert a.tolist() == b.tolist()
            spilled += int(a[2])
        try:
            sh.plan()
        except N.MagicPigError as e:
            assert "dense KV cache is full" in str(e)
            break
        tw.plan()
        steps += 1
        q = torch.randn((3, Hq, d), generator=gen).bfloat16().to(DEV)
        k = torch.randn((3, Hkv, d), generator=gen).bfloat16().to(DEV)
        assert torch.equal(sh.decode(1, q, k, k), tw.decode(1, q, k, k))
        for c in (sh, tw):
            c.dense_decode(0, q, k, k)
        a, b = sh.last_out_f32(), tw.last_out_f32()
        assert torch.allclose(a, b, rtol=0, atol=TOL)
    assert steps == R and spilled > 0
    assert sh.error_flags() == 0


def test_memory(cuda_lib):
    B, C, Hq, Hkv, K, L, M, R = 4, 1, 8, 2, 8, 60, 4096, 48
    hf = synth.make_hash_func(d, K, L, seed=1)
    plain, shared = make_ctx(B, C, Hq, Hkv, M, K, L, hf), make_ctx(B, C, Hq, Hkv, M, K, L, hf, R=R)
    rec = 2 * d * 2
    per_layer = C * Hkv * M * rec + B * Hkv * R * rec - B * Hkv * M * rec   # one dense layer
    assert shared.device_bytes - plain.device_bytes == per_layer + max(B * 4, 16)
    assert shared.get_info("dense_tail_rows") == R and plain.get_info("dense_tail_rows") == 0


def test_b8_one_dense_prompt_copy(cuda_lib):
    """B = 8 over one slot at a C2-size dense shape (Hkv = 8, M = 98 304, two dense layers): one prompt copy instead of eight."""
    B, Hq, Hkv, M, R = 8, 32, 8, 98304, 264
    hf = synth.make_hash_func(d, 10, 150, seed=4)

    def ctx_for(R_):
        c = Context(10, 150, 3, Hq, Hkv, d, B, M, NS, NL, GEN, dense_layers=[0, 1], alloc_dense_kv=True, device=DEV, num_contexts=1,
                    dense_tail_rows=R_)
        c.set_hash_func(hf.to(DEV))
        return c

    plain = ctx_for(0)
    plain_bytes = plain.device_bytes
    del plain
    torch.cuda.empty_cache()
    shared = ctx_for(R)
    rec = 2 * d * 2
    assert plain_bytes - shared.device_bytes == 2 * ((B - 1) * Hkv * M * rec - B * Hkv * R * rec) - 32
    P = 98000
    g = torch.Generator(device=DEV).manual_seed(5)
    for layer in (0, 1):
        kk = torch.randn((P, Hkv, d), generator=g, device=DEV).bfloat16()
        shared.dense_fill(layer, 0, kk, kk, P)
    for b in range(1, B):
        shared.fork(0, b)
    q = torch.randn((B, Hq, d), generator=g, device=DEV).bfloat16()
    k = torch.randn((B, Hkv, d), generator=g, device=DEV).bfloat16()
    k[:] = k[0]
    q[:] = q[0]
    shared.set_option("out_f32", 1)
    shared.plan()
    shared.dense_decode(0, q, k, k)
    o = shared.last_out_f32().reshape(B, Hq, d)
    assert torch.isfinite(o).all()
    assert torch.allclose(o, o[0:1].expand_as(o), rtol=0, atol=TOL)   # same prompt, same new row: same output


def test_refusals(cuda_lib):
    hf = synth.make_hash_func(d, 8, 60, seed=1)
    with pytest.raises(N.MagicPigError, match="fewer context slots"):
        make_ctx(4, 0, 8, 2, 512, 8, 60, hf, R=16)
    with pytest.raises(N.MagicPigError, match="fewer context slots"):
        make_ctx(4, 4, 8, 2, 512, 8, 60, hf, R=16)
    with pytest.raises(N.MagicPigError, match="alloc_dense_kv"):
        Context(8, 60, 2, 8, 2, d, 4, 512, NS, NL, GEN, dense_layers=[0], alloc_dense_kv=False, device=DEV, num_contexts=1,
                dense_tail_rows=16)
    for R in (-1, 513):
        with pytest.raises(N.MagicPigError, match="outside"):
            make_ctx(4, 1, 8, 2, 512, 8, 60, hf, R=R)
    c = make_ctx(4, 1, 8, 2, 512, 8, 60, hf, R=16)
    c.set_option("dense_impl", 0)
    q = torch.zeros((4, 8, d), dtype=torch.bfloat16, device=DEV)
    k = torch.zeros((4, 2, d), dtype=torch.bfloat16, device=DEV)
    c.plan()
    with pytest.raises(N.MagicPigError, match="dense_impl"):
        c.dense_decode(0, q, k, k)


def test_dropin_server(cuda_lib):
    from magicpig_b200.attnserver import LSHSparseAttnServer
    cfg = _Cfg()
    cfg.num_hidden_layers, cfg.num_key_value_heads, cfg.num_attention_heads, cfg.hidden_size = 3, 2, 8, 8 * d
    B, P = 3, 1200
    hf = torch.randn((d, 8 * 60), generator=torch.Generator().manual_seed(2)).bfloat16()
    mk = lambda C, R: LSHSparseAttnServer(cfg, K=8, L=60, batch_size=B, max_length=2048, dense_layers=(0,), device=DEV,  # noqa: E731
                                          hash_func=hf, generation_buffer=16, num_contexts=C, dense_tail_rows=R)
    sh, tw = mk(1, 24), mk(None, None)
    assert sh.ctx.dense_tail_rows == 24 and tw.ctx.dense_tail_rows == 0
    g = torch.Generator().manual_seed(3)
    kv = [(torch.randn((P, 2, d), generator=g).bfloat16().to(DEV), torch.randn((P, 2, d), generator=g).bfloat16().to(DEV)) for _ in range(3)]
    for srv, reqs in ((sh, [0]), (tw, range(B))):
        srv.alloc_buffer(P)
        for layer in range(3):
            for b in reqs:
                srv.fill(layer, b, kv[layer][0], kv[layer][1], P)
                srv.build_table(layer, b, P)
    sh.fork(0, [1, 2])
    for c in (sh, tw):
        c.ctx.set_option("out_f32", 1)
    for _ in range(4):
        q = torch.randn((B, 8, 1, d), generator=g).bfloat16().to(DEV)
        k = torch.randn((B, 2, 1, d), generator=g).bfloat16().to(DEV)
        for srv in (sh, tw):
            srv.plan()
        sh.decode(q, k, k, 0)
        tw.decode(q, k, k, 0)
        assert torch.allclose(sh.ctx.last_out_f32(), tw.ctx.last_out_f32(), rtol=0, atol=TOL)
        for layer in (1, 2):
            assert torch.equal(sh.decode(q, k, k, layer), tw.decode(q, k, k, layer))


def test_runner_shared_dense(cuda_lib):
    """Captured steps of the runner with R > 0 against R = 0 (both over one slot): the logits differ only through the dense layers'
    summation order, which flips bf16 roundings of their outputs; the random-weight layers after them amplify that to at most 0.25
    absolute on logits of magnitude ~2, and the argmax tokens are equal."""
    from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner
    runs = []
    for R in (64, None):
        r = LlamaDecodeRunner(LLAMA31_8B, 8, 60, 3, 4096, device=DEV, num_layers=3, num_contexts=1, dense_tail_rows=R,
                              dense_layers=(0, 2))
        r.synthetic_prefill(3000, shared=True)
        r.ids.copy_(torch.tensor([[11], [22], [33]], device=DEV))
        r.capture()
        runs.append(r)
    assert runs[0].server.ctx.dense_tail_rows == 64 and runs[1].server.ctx.dense_tail_rows == 0
    assert runs[0].server.ctx.device_bytes < runs[1].server.ctx.device_bytes
    for _ in range(3):
        a, b = runs[0].replay().clone(), runs[1].replay().clone()
        torch.cuda.synchronize()
        assert torch.allclose(a, b, rtol=0, atol=0.25), (a - b).abs().max().item()
        assert torch.equal(a.argmax(-1), b.argmax(-1))
