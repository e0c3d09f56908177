"""Context slots (`-m gpu`): several requests of a batch decode over one sampled store and one set of hash tables.

Every check compares a context with fewer slots than requests (filled once, then fork / bind) against a twin with one slot per
request, each filled with the same data, given the same per-request q / k / v:
  * fork twin: single-token, T-token (with rewind) and tree (with accept) steps give bitwise equal codes, nnz, index lists, fp32
    and bf16 outputs on four fused shapes, fused_kreg 0 / 1 and the host-buffer entry point; the three-launch path is within
    1e-5; a forked request is within 1e-3 of the oracle; dense layers are equal;
  * two documents on two slots, a refill through one request, bind, a step captured before fork / bind;
  * spill of an exclusive request on a slot other than its index, of two exclusive requests whose slots are in the reverse of
    their request order, refused spills of shared requests, refused calls;
  * memory: one slot less is the per-slot bytes less; B = 8 on one C2-size context;
  * the drop-in class and the Llama runner.
"""
import ctypes

import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200 import synth
from magicpig_b200.ops import Context
from tests.support.fp64 import assert_1e3_f32, oracle_decode
from tests.support.library import (DEV, NL, NS, Doc, _Cfg, assert_lists_equal, assert_tables_equal, d, lsh_tables,
                                   two_layer_context)

pytestmark = pytest.mark.gpu
GEN = 32


def make_ctx(B, C, Hq, Hkv, M, K, L, hf, impl=1, kreg=0, t_max=1, gen=GEN):
    return two_layer_context(K, L, Hq, Hkv, B, M, gen, hf, dict(decode_impl=impl, fused_kreg=kreg, out_f32=1, save_mask=1),
                             alloc_dense_kv=True, max_query_tokens=t_max, num_contexts=C)


class Pair:
    """A shared context (documents filled through their source requests, then forked) and its twin (every request filled)."""

    def __init__(self, B, C, Hq, Hkv, n, K, L, docs_of, forks, seed=0, impl=1, kreg=0, t_max=1, fill=None):
        self.B, self.Hq, self.Hkv, self.G = B, Hq, Hkv, Hq // Hkv
        self.hf = synth.make_hash_func(d, K, L, seed=seed + 11)
        M = n + 256
        self.docs = {i: Doc(Hkv, n, K, L, self.hf, seed + 100 * (i + 1)) for i in set(docs_of)}
        self.docs_of = list(docs_of)   # document of each request
        self.sh = make_ctx(B, C, Hq, Hkv, M, K, L, self.hf, impl, kreg, t_max)
        self.tw = make_ctx(B, 0, Hq, Hkv, M, K, L, self.hf, impl, kreg, t_max)
        dsts = {dst for _, dst in forks}
        for b in (fill if fill is not None else [b for b in range(B) if b not in dsts]):
            self.docs[docs_of[b]].fill_store(self.sh, b)
            self.docs[docs_of[b]].fill_request(self.sh, b)
        for src, dst in forks:
            self.sh.fork(src, dst)
        for b in range(B):
            self.docs[docs_of[b]].fill_store(self.tw, b)
            self.docs[docs_of[b]].fill_request(self.tw, b)
        self.g = torch.Generator().manual_seed(seed + 7)

    def qkv(self, T=1):
        B, Hq, Hkv, g = self.B, self.Hq, self.Hkv, self.g
        return (torch.randn((B, T, Hq, d), generator=g).bfloat16().to(DEV), torch.randn((B, T, Hkv, d), generator=g).bfloat16().to(DEV),
                torch.randn((B, T, Hkv, d), generator=g).bfloat16().to(DEV))

    def compare_probe(self, exact_out=True, tol=None):
        assert_lists_equal(*self.sh.last_probe(True), *self.tw.last_probe(True))
        if self.sh.get_info("last_decode_fused"):
            assert torch.equal(self.sh.last_codes(), self.tw.last_codes()), "codes differ"
        oa, ob = self.sh.last_out_f32(), self.tw.last_out_f32()
        if exact_out:
            assert torch.equal(oa, ob), f"fp32 outputs differ (max {(oa - ob).abs().max().item()})"
        else:
            assert torch.allclose(oa, ob, rtol=0, atol=tol), f"fp32 outputs differ by {(oa - ob).abs().max().item()}"

    def single(self, exact_out=True, tol=None, hook=None):
        q, k, v = self.qkv()
        outs = []
        for ctx in (self.sh, self.tw):
            ctx.plan()
            outs.append(ctx.decode(1, q[:, 0], k[:, 0], v[:, 0]).clone())
        self.compare_probe(exact_out, tol)
        if hook:
            hook(q, k, v)
        if exact_out:
            assert torch.equal(outs[0], outs[1])
        qd, kd, vd = self.qkv()
        dense = [ctx.dense_decode(0, qd[:, 0], kd[:, 0], vd[:, 0]).clone() for ctx in (self.sh, self.tw)]
        assert torch.equal(dense[0], dense[1]), "dense layer differs"
        return q, k, v

    def tokens(self, T, drop):
        q, k, v = self.qkv(T)
        dr = torch.tensor(drop, dtype=torch.int32, device=DEV)
        outs = []
        for ctx in (self.sh, self.tw):
            ctx.plan(T)
            outs.append(ctx.decode_tokens(1, T, q, k, v).clone())
        self.compare_probe()
        assert torch.equal(outs[0], outs[1])
        qd, kd, vd = self.qkv(T)
        dense = [ctx.dense_decode_tokens(0, T, qd, kd, vd).clone() for ctx in (self.sh, self.tw)]
        assert torch.equal(dense[0], dense[1])
        for ctx in (self.sh, self.tw):
            ctx.rewind(dr)

    def tree(self, parents, nodes, count):
        T = len(parents)
        par = torch.tensor([parents] * self.B, dtype=torch.int32, device=DEV)
        q, k, v = self.qkv(T)
        outs = []
        for ctx in (self.sh, self.tw):
            ctx.plan(T, parents=par)
            outs.append(ctx.decode_tokens(1, T, q, k, v).clone())
        self.compare_probe()
        assert torch.equal(outs[0], outs[1])
        qd, kd, vd = self.qkv(T)
        for ctx in (self.sh, self.tw):
            ctx.dense_decode_tokens(0, T, qd, kd, vd)
        nd = torch.tensor([nodes + [0] * (T - len(nodes))] * self.B, dtype=torch.int32, device=DEV)
        ct = torch.tensor(count, dtype=torch.int32, device=DEV)
        for ctx in (self.sh, self.tw):
            ctx.accept(nd, ct)


# B = 4 on four fused shapes: clusters of several CTAs, two key segments, one CTA per head, two CTAs per SM
FUSED_SHAPES = [(8, 2, 1500, 8, 60), (2, 1, 70000, 8, 40), (32, 8, 2000, 8, 60), (40, 8, 1200, 8, 40)]


@pytest.mark.parametrize("kreg", [0, 1])
@pytest.mark.parametrize("Hq,Hkv,n,K,L", FUSED_SHAPES)
def test_fork_twin(cuda_lib, Hq, Hkv, n, K, L, kreg):
    B = 4
    p = Pair(B, 1, Hq, Hkv, n, K, L, [0] * B, [(0, 1), (0, 2), (0, 3)], seed=Hq + n, kreg=kreg, t_max=4)
    assert p.sh.num_contexts == 1 and p.tw.num_contexts == B
    doc = p.docs[0]

    def oracle_check(q, k, v):   # the forked requests against the oracle fed the shared store and their own (forked) window
        t = dict(B=B, Hq=Hq, Hkv=Hkv, d=d, K=K, L=L, n=n, M=n + 256, hash_func=p.hf, kcodes=doc.kcodes[None].expand(B, -1, -1, -1),
                 key=doc.key[None].expand(B, -1, -1, -1), value=doc.value[None].expand(B, -1, -1, -1),
                 key_norm=doc.kn[None].expand(B, -1, -1), avg_k=doc.avg.reshape(1, Hkv, 1, d).expand(B, -1, -1, -1))
        wk = doc.wk[None].expand(B, -1, -1, -1)
        wv = doc.wv[None].expand(B, -1, -1, -1)
        _, nz_ref, _, o_exact = oracle_decode(t, q[:, 0].cpu().reshape(B, Hq, 1, d), k[:, 0].cpu().reshape(B, Hkv, 1, d),
                                              v[:, 0].cpu().reshape(B, Hkv, 1, d), wk, wv, Hq // Hkv)
        assert torch.equal(p.sh.last_probe()[0].cpu(), nz_ref)
        assert_1e3_f32(p.sh.last_out_f32().cpu(), o_exact)

    p.single(hook=oracle_check)
    p.single()
    p.tokens(3, [0, 1, 2, 3])
    p.tree([-1, 0, 0, 1], [0, 2], [2, 1, 0, 2])
    p.single()
    # the host-buffer entry point
    q, k, v = p.qkv()
    outs = []
    for ctx in (p.sh, p.tw):
        ctx.plan()
        o = torch.zeros((B, Hq * d), dtype=torch.bfloat16).pin_memory()
        ctx.decode_host(1, q[:, 0].cpu().contiguous().pin_memory(), k[:, 0].cpu().contiguous().pin_memory(),
                        v[:, 0].cpu().contiguous().pin_memory(), o)
        outs.append(o)
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(p.sh.last_out_f32(), p.tw.last_out_f32())


def test_fork_twin_three_launch(cuda_lib):
    p = Pair(4, 1, 8, 2, 1500, 8, 60, [0] * 4, [(0, 1), (0, 2), (0, 3)], seed=5, impl=0)
    for _ in range(3):
        p.single(exact_out=False, tol=1e-5)


def test_two_documents_and_refill(cuda_lib):
    # slot 0 <- document 0 through request 0, slot 1 <- document 1 through request 1; 0 -> 2 and 1 -> 3 forked
    p = Pair(4, 2, 8, 2, 1500, 8, 60, [0, 1, 0, 1], [(0, 2), (1, 3)], seed=9)
    p.single()
    p.single()
    # a refill through request 0 changes the context of requests 0 and 2 only
    new = Doc(2, 1500, 8, 60, p.hf, 777)
    new.fill_store(p.sh, 0)
    new.fill_store(p.tw, 0)
    new.fill_store(p.tw, 2)
    p.single()
    p.single()


def test_bind(cuda_lib):
    # B = 3, C = 2: request 2 starts on slot 0, is bound to slot 1, which is filled through it, then gets its window
    p = Pair(3, 2, 8, 2, 1500, 8, 60, [0, 1, 1], [], seed=13, fill=[0, 1])
    p.sh.bind(2, 1)
    p.docs[1].fill_store(p.sh, 2)
    p.docs[1].fill_request(p.sh, 2)
    for _ in range(3):
        p.single()
    with pytest.raises(N.MagicPigError):
        p.sh.bind(0, 2)      # slot out of range
    with pytest.raises(N.MagicPigError):
        p.sh.bind(3, 0)      # request out of range
    with pytest.raises(N.MagicPigError):
        p.tw.bind(0, 1)      # every request owns its slot


def test_graph_replays_new_bindings(cuda_lib):
    # two identical shared contexts (B = 3, C = 2): one replays a step captured before a fork and a bind, the other runs eagerly
    hf = synth.make_hash_func(d, 8, 60, seed=3)
    docs = [Doc(2, 1500, 8, 60, hf, 300 + i) for i in range(2)]
    ctxs = []
    for _ in range(2):
        c = make_ctx(3, 2, 8, 2, 1756, 8, 60, hf)
        docs[0].fill_store(c, 0); docs[0].fill_request(c, 0); docs[0].fill_request(c, 2)
        docs[1].fill_store(c, 1); docs[1].fill_request(c, 1)
        ctxs.append(c)
    g_ctx, e_ctx = ctxs
    q = torch.zeros((3, 8, d), dtype=torch.bfloat16, device=DEV)
    k = torch.zeros((3, 2, d), dtype=torch.bfloat16, device=DEV)
    v = torch.zeros_like(k)
    out = torch.zeros((3, 8 * d), dtype=torch.bfloat16, device=DEV)
    for c in ctxs:   # warm-up (launch plans, function attributes) outside the capture, on both
        c.plan()
        c.decode(1, q, k, v)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        g_ctx.plan()
        g_ctx.decode(1, q, k, v, out)
    gen = torch.Generator().manual_seed(5)

    def step():
        q.copy_(torch.randn((3, 8, d), generator=gen).bfloat16())
        k.copy_(torch.randn((3, 2, d), generator=gen).bfloat16())
        v.copy_(torch.randn((3, 2, d), generator=gen).bfloat16())
        graph.replay()
        torch.cuda.synchronize()
        e_ctx.plan()
        ref = e_ctx.decode(1, q, k, v)
        assert torch.equal(out, ref)
        assert torch.equal(g_ctx.last_probe()[0], e_ctx.last_probe()[0])

    step()
    for c in ctxs:
        c.fork(1, 2)          # request 2 moves from slot 0 to slot 1
    step()
    for c in ctxs:
        c.bind(0, 1)          # request 0 now reads document 1 through its own window
    step()


def twin_step(sh, tw, gen):
    """One single-token step of a context with slots and its twin on the same random q / k / v: bitwise equal outputs and nnz."""
    q = torch.randn((sh.B, sh.Hq, d), generator=gen).bfloat16().to(DEV)
    k = torch.randn((sh.B, sh.Hkv, d), generator=gen).bfloat16().to(DEV)
    v = torch.randn((sh.B, sh.Hkv, d), generator=gen).bfloat16().to(DEV)
    outs = []
    for c in (sh, tw):
        c.plan()
        outs.append(c.decode(1, q, k, v).clone())
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(sh.last_probe()[0], tw.last_probe()[0])


def test_spill_exclusive_and_refused(cuda_lib):
    K, L, n, Hq, Hkv = 8, 60, 1500, 8, 2
    hf = synth.make_hash_func(d, K, L, seed=17)
    short = Doc(Hkv, n, K, L, hf, 500, w=NS + 8)     # requests 0 and 1 share slot 0 and never reach a spill
    long_ = Doc(Hkv, n, K, L, hf, 600, w=NS + NL + 6)
    sh = make_ctx(3, 2, Hq, Hkv, n + 256, K, L, hf)
    tw = make_ctx(3, 0, Hq, Hkv, n + 256, K, L, hf)
    sh.bind(1, 0)
    sh.bind(2, 1)            # request 2 alone on slot 1
    short.fill_store(sh, 0); short.fill_request(sh, 0); short.fill_request(sh, 1)
    long_.fill_store(sh, 2); long_.fill_request(sh, 2)
    for b, doc in ((0, short), (1, short), (2, long_)):
        doc.fill_store(tw, b); doc.fill_request(tw, b)
    gen = torch.Generator().manual_seed(3)
    for _ in range(4):
        twin_step(sh, tw, gen)
    assert sh.spill_window().tolist() == [0, 0, 10] == tw.spill_window().tolist()
    # the slot's tables equal a device rebuild over the keys the slot now stores
    k_st = sh.read_cache(1, True, False, False)[0]
    ref = Context(K, L, 2, Hq, Hkv, d, 1, n + 256, NS, NL, 8, dense_layers=[0], device=DEV)
    ref.set_hash_func(hf.to(DEV))
    ref.lsh_build(1, 0, sh.hash_keys(k_st[1, :, : n + 10].contiguous()))
    o, i = lsh_tables(sh, 1)
    ro, ri = lsh_tables(ref, 1)
    assert_tables_equal((o[1], i[1]), (ro[0], ri[0]))
    for _ in range(3):
        twin_step(sh, tw, gen)
    # a request that would spill into a slot another non-empty request reads is refused, and nothing changes
    shr = make_ctx(2, 1, Hq, Hkv, n + 256, K, L, hf)
    ref2 = make_ctx(2, 1, Hq, Hkv, n + 256, K, L, hf)
    for c in (shr, ref2):
        long_.fill_store(c, 0); long_.fill_request(c, 0); c.fork(0, 1)
    for c in (shr, ref2):
        c.plan()
        c.decode(1, *(torch.ones((2, h, d), dtype=torch.bfloat16, device=DEV) for h in (Hq, Hkv, Hkv)))
    before = lsh_tables(shr, 1), shr.read_cache(1)
    with pytest.raises(N.MagicPigError, match="shares"):
        shr.spill_window()
    after = lsh_tables(shr, 1), shr.read_cache(1)
    assert all(torch.equal(a, b) for a, b in zip(before[0], after[0]))
    assert all(torch.equal(a, b) for a, b in zip(before[1], after[1]))
    q = torch.randn((2, Hq, d), generator=gen).bfloat16().to(DEV)
    kv = torch.randn((2, Hkv, d), generator=gen).bfloat16().to(DEV)
    outs = []
    for c in (shr, ref2):      # windows and lengths unchanged: the next decode equals a context that never tried to spill
        c.plan()
        outs.append(c.decode(1, q, kv, kv).clone())
    assert torch.equal(outs[0], outs[1])


def test_spill_exclusive_slots_out_of_request_order(cuda_lib):
    # B = 4, C = 3: request 0 alone on slot 2, request 3 alone on slot 0, requests 1 and 2 share slot 1 with short windows; the
    # two spilling requests spill different row counts, and slot order differs from request order
    K, L, n, Hq, Hkv = 8, 60, 1500, 8, 2
    hf = synth.make_hash_func(d, K, L, seed=19)
    short = Doc(Hkv, n, K, L, hf, 700, w=NS + 8)
    docs = [Doc(Hkv, n, K, L, hf, 800, w=NS + NL + 6), short, short, Doc(Hkv, n, K, L, hf, 900, w=NS + NL + 13)]
    sh = make_ctx(4, 3, Hq, Hkv, n + 256, K, L, hf)
    tw = make_ctx(4, 0, Hq, Hkv, n + 256, K, L, hf)
    sh.bind(0, 2)
    sh.bind(2, 1)
    for b in (0, 3, 1):
        docs[b].fill_store(sh, b)
    for b in range(4):
        docs[b].fill_request(sh, b)
        docs[b].fill_store(tw, b); docs[b].fill_request(tw, b)
    gen = torch.Generator().manual_seed(5)
    for _ in range(4):
        twin_step(sh, tw, gen)
    assert sh.spill_window().tolist() == [10, 0, 0, 17] == tw.spill_window().tolist()
    # slot 2 holds request 0's keys, slot 0 request 3's, slot 1 the prompt alone: the records and norms of the twin's request,
    # and tables equal to a rebuild over the stored keys
    cache_sh, cache_tw = sh.read_cache(1), tw.read_cache(1)
    o, i = lsh_tables(sh, 1)
    ref = Context(K, L, 2, Hq, Hkv, d, 1, n + 256, NS, NL, 8, dense_layers=[0], device=DEV)
    ref.set_hash_func(hf.to(DEV))
    for c, b, g in ((2, 0, 10), (0, 3, 17), (1, 1, 0)):
        for a, t in zip(cache_sh, cache_tw):
            assert torch.equal(a[c, :, : n + g], t[b, :, : n + g]), f"slot {c}: stored records differ"
        ref.lsh_build(1, 0, sh.hash_keys(cache_sh[0][c, :, : n + g].contiguous()))
        ro, ri = lsh_tables(ref, 1)
        assert_tables_equal((o[c], i[c]), (ro[0], ri[0]))
    for _ in range(3):
        twin_step(sh, tw, gen)


def test_config_and_option_refusals(cuda_lib, monkeypatch):
    """mpig_create refuses ctas_per_sm outside {0, 1, 2} and a non-zero reserved field; option keys that select nothing are
    unknown keys."""
    hf = synth.make_hash_func(d, 6, 24, seed=1)
    for v in ("3", "-1"):
        monkeypatch.setenv("MPIG_CTA_PER_SM", v)
        with pytest.raises(N.MagicPigError, match="ctas_per_sm"):
            make_ctx(3, 1, 4, 4, 400, 6, 24, hf)
    monkeypatch.delenv("MPIG_CTA_PER_SM")
    ctx = make_ctx(3, 1, 4, 4, 400, 6, 24, hf)
    for key in ("attend_stages", "keyhash_stages", "attend_impl"):
        with pytest.raises(N.MagicPigError, match="unknown key"):
            ctx.set_option(key, 1)
    cfg = N.MpigConfig(abi_version=N.MPIG_ABI_VERSION, device=torch.device(DEV).index or 0, K=6, L=24, num_layers=1,
                       num_attention_heads=4, num_key_value_heads=4, head_dim=d, batch_size=3, max_length=400)
    h = ctypes.c_void_p()
    assert cuda_lib.mpig_create(ctypes.byref(cfg), ctypes.byref(h)) == N.MPIG_OK
    cuda_lib.mpig_destroy(h)
    for i in range(4):
        cfg.reserved[i] = 1
        assert cuda_lib.mpig_create(ctypes.byref(cfg), ctypes.byref(h)) == -1   # MPIG_EINVAL
        assert f"reserved[{i}]".encode() in cuda_lib.mpig_last_error()
        cfg.reserved[i] = 0


def test_refusals(cuda_lib):
    hf = synth.make_hash_func(d, 6, 24, seed=1)
    for C in (-1, 4):
        with pytest.raises(N.MagicPigError, match="num_contexts"):
            make_ctx(3, C, 4, 4, 400, 6, 24, hf)
    ctx = make_ctx(3, 1, 4, 4, 400, 6, 24, hf, t_max=2)
    doc = Doc(4, 100, 6, 24, hf, 2)
    doc.fill_store(ctx, 0); doc.fill_request(ctx, 0)
    for src, dst in ((0, 0), (-1, 1), (0, 3), (3, 0)):
        with pytest.raises(N.MagicPigError):
            ctx.fork(src, dst)
    # a fork ends the pending step: rewind and accept are refused until the next plan
    ctx.plan(2)
    ctx.fork(0, 1)
    with pytest.raises(N.MagicPigError):
        ctx.rewind(torch.zeros(3, dtype=torch.int32, device=DEV))
    ctx.pending_tokens = 2
    with pytest.raises(N.MagicPigError):
        ctx.accept(torch.zeros((3, 2), dtype=torch.int32, device=DEV), torch.ones(3, dtype=torch.int32, device=DEV))
    ctx.plan(2)
    ctx.bind(2, 0)
    with pytest.raises(N.MagicPigError):
        ctx.rewind(torch.zeros(3, dtype=torch.int32, device=DEV))
    ctx.plan(2)
    ctx.rewind(torch.zeros(3, dtype=torch.int32, device=DEV))


def test_memory_per_slot(cuda_lib):
    B, Hq, Hkv, K, L, M = 4, 8, 2, 8, 60, 4096
    hf = synth.make_hash_func(d, K, L, seed=1)
    full, one = make_ctx(B, 0, Hq, Hkv, M, K, L, hf), make_ctx(B, 1, Hq, Hkv, M, K, L, hf)
    S, NB = full.get_info("table_segments"), 1 << K
    per_slot = Hkv * M * 2 * d * 2 + Hkv * M * 4 + Hkv * L * S * (NB + 1) * 4 + Hkv * L * M * 2   # one sparse layer
    assert full.device_bytes - one.device_bytes == (B - 1) * per_slot


def test_c2_size_b8_one_context(cuda_lib):
    """B = 8 requests over ONE C2-size context (n = 97 932, K10 L150) on two sparse layers: per-request nnz and index lists equal
    those of a twin that holds eight copies."""
    B, Hq, Hkv, K, L, n = 8, 32, 8, 10, 150, 97932
    hf = synth.make_hash_func(d, K, L, seed=4)
    docs = [Doc(Hkv, n, K, L, hf, 40 + l, on_gpu=True) for l in range(2)]

    def ctx_for(C):
        c = Context(K, L, 3, Hq, Hkv, d, B, n + 368, NS, NL, GEN, dense_layers=[0], device=DEV, num_contexts=C)
        c.set_option("save_mask", 1)
        c.set_hash_func(hf.to(DEV))
        return c

    sh, tw = ctx_for(1), ctx_for(0)
    gen = torch.Generator().manual_seed(8)
    wins = [(torch.randn((Hkv, NS + NL, d), generator=gen).bfloat16().to(DEV),
             torch.randn((Hkv, NS + NL, d), generator=gen).bfloat16().to(DEV)) for _ in range(2)]
    avg = torch.zeros((Hkv, d), dtype=torch.bfloat16, device=DEV)
    for c, reqs in ((sh, [0]), (tw, range(B))):
        for layer, doc in zip((1, 2), docs):
            codes = c.hash_keys(doc.key)
            for b in reqs:
                c.attn_fill(layer, b, doc.key, doc.value, doc.kn)
                c.lsh_build(layer, b, codes)
                c.window_fill(layer, b, avg, *wins[layer - 1])
    for b in range(1, B):
        sh.fork(0, b)
    assert sh.device_bytes < tw.device_bytes
    for _ in range(2):
        q = torch.randn((B, Hq, d), generator=gen).bfloat16().to(DEV)
        k = torch.randn((B, Hkv, d), generator=gen).bfloat16().to(DEV)
        for c in (sh, tw):
            c.plan()
        for layer in (1, 2):
            outs = []
            for c in (sh, tw):
                outs.append(c.decode(layer, q, k, k).clone())
            assert_lists_equal(*sh.last_probe(True), *tw.last_probe(True))
            assert torch.equal(outs[0], outs[1])


def test_dropin_fork(cuda_lib):
    from magicpig_b200.attnserver import LSHSparseAttnServer
    cfg = _Cfg()
    cfg.num_hidden_layers, cfg.num_key_value_heads, cfg.num_attention_heads, cfg.hidden_size = 3, 2, 8, 8 * d
    B, P = 3, 1200
    hf = torch.randn((d, 8 * 60), generator=torch.Generator().manual_seed(2)).bfloat16()
    mk = lambda C: LSHSparseAttnServer(cfg, K=8, L=60, batch_size=B, max_length=2048, dense_layers=(0,), device=DEV,  # noqa: E731
                                       hash_func=hf, generation_buffer=16, num_contexts=C)
    sh, tw = mk(1), mk(None)
    g = torch.Generator().manual_seed(3)
    kv = [(torch.randn((P, 2, d), generator=g).bfloat16().to(DEV), torch.randn((P, 2, d), generator=g).bfloat16().to(DEV)) for _ in range(3)]
    for srv, reqs in ((sh, [0]), (tw, range(B))):
        srv.alloc_buffer(P)
        for layer in range(3):
            for b in reqs:
                srv.fill(layer, b, kv[layer][0], kv[layer][1], P)
                srv.build_table(layer, b, P)
    sh.fork(0, [1, 2])
    for layer in range(3):
        assert torch.equal(sh.avg_k[layer], tw.avg_k[layer])
    for _ in range(4):
        q = torch.randn((B, 8, 1, d), generator=g).bfloat16().to(DEV)
        k = torch.randn((B, 2, 1, d), generator=g).bfloat16().to(DEV)
        for srv in (sh, tw):
            srv.plan()
        for layer in range(3):
            assert torch.equal(sh.decode(q, k, k, layer), tw.decode(q, k, k, layer))


def test_runner_shared(cuda_lib):
    from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner
    runs = []
    for C in (1, None):
        r = LlamaDecodeRunner(LLAMA31_8B, 8, 60, 3, 4096, device=DEV, num_layers=3, num_contexts=C)
        r.synthetic_prefill(3000, shared=True)
        r.ids.copy_(torch.tensor([[11], [22], [33]], device=DEV))
        r.capture()
        runs.append(r)
    assert runs[0].server.ctx.num_contexts == 1 and runs[1].server.ctx.num_contexts == 3
    for _ in range(3):
        a, b = runs[0].replay().clone(), runs[1].replay().clone()
        torch.cuda.synchronize()
        assert torch.equal(a, b)
    # fork of the runner copies the position too
    runs[0].fork(0, 2)
    assert runs[0].pos[2].item() == runs[0].pos[0].item()
