"""Shared spill (`-m gpu`): requests that share a context slot spill their windows into it, and each sees only its own spilled keys.

A context created with shared_spill=True and fewer slots than requests is compared against a twin in which every request owns its
slot and was filled with the same document, given the same per-request q / k / v and the same spills.  A request of the shared
context must then sample exactly what its twin samples: equal codes and nnz, equal index lists once the shared slot's keys are
renumbered into the twin's (prompt keys unchanged, the private keys the request sees in time order after them), and fp32
outputs within 1e-5 of the twin's largest output (the order of the sampled keys, and so the summation order, differs).
Covered: the fused kernel (fused_kreg 0 / 1, 512-thread CTAs, several selection passes, with and without the saved lists), the
host-buffer entry point, the three-launch path, T-token chains with rewind and trees with accept, a geometry whose key segments
split the requests' private keys, the slot's tables after a spill of several requests, fork and bind, graph replay across a
spill, a fork and a bind, the refusals, the drop-in class and the Llama runner.
"""
import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200 import synth
from magicpig_b200.ops import Context
from tests.support.fp64 import assert_1e3_f32, oracle_decode
from tests.support.library import DEV, NL, NS, Doc, _Cfg, assert_tables_equal, d, lsh_tables, two_layer_context

pytestmark = pytest.mark.gpu
GEN = 32
Hq, Hkv, K, L, M = 8, 2, 8, 60, 4096


def make_ctx(B, C, hf, shared, impl=1, kreg=0, selcap=2048, save_mask=1):
    return two_layer_context(K, L, Hq, Hkv, B, M, GEN, hf, dict(decode_impl=impl, fused_kreg=kreg, fused_selcap=selcap, out_f32=1,
                                                                save_mask=save_mask),
                             max_query_tokens=4, num_contexts=C, shared_spill=shared)


class Model:
    """Host model of the shared context's private keys: per slot the offsets handed out so far, per request its slot and the
    offsets it sees (ascending = time order)."""

    def __init__(self, B, C, n):
        self.n, self.slot = n, [b % C for b in range(B)]
        self.count = [0] * C
        self.vis = [[] for _ in range(B)]

    def spill(self, g):
        for b, gb in enumerate(g):   # a slot's new keys go in request order
            c = self.slot[b]
            self.vis[b] += range(self.count[c], self.count[c] + gb)
            self.count[c] += gb

    def fork(self, src, dst):
        self.slot[dst], self.vis[dst] = self.slot[src], list(self.vis[src])

    def bind(self, r, c):
        self.slot[r], self.vis[r] = c, []

    def refill(self, c):
        self.count[c] = 0
        for b in range(len(self.slot)):
            if self.slot[b] == c:
                self.vis[b] = []

    def key_map(self, b):
        """shared slot key -> twin key for request b (-1: a key b must not see)"""
        mp = torch.full((M,), -1, dtype=torch.long, device=DEV)
        mp[: self.n] = torch.arange(self.n, device=DEV)
        if self.vis[b]:
            mp[self.n + torch.tensor(self.vis[b], device=DEV)] = self.n + torch.arange(len(self.vis[b]), device=DEV)
        return mp


def compare(sh, tw, model, lists=True):
    B = sh.B
    nz_s, res_s = sh.last_probe(lists)
    nz_t, res_t = tw.last_probe(lists)
    assert torch.equal(nz_s, nz_t), "nnz differ"
    if lists:
        if sh.get_info("last_decode_fused"):
            assert torch.equal(sh.last_codes(), tw.last_codes()), "codes differ"
        per = nz_s.shape[0] // B
        valid = torch.arange(M, device=DEV)[None] < nz_s[:, None]
        for b in range(B):
            r = slice(b * per, (b + 1) * per)
            mapped = model.key_map(b)[res_s[r].clamp(0, M - 1).long()]
            assert bool((mapped[valid[r]] >= 0).all()), f"request {b} sampled a private key it does not see"
            assert torch.equal(torch.where(valid[r], mapped, -1), torch.where(valid[r], res_t[r].long(), -1)), f"request {b}: lists differ"
    oa, ob = sh.last_out_f32(), tw.last_out_f32()
    err = float((oa - ob).abs().max())
    assert err <= 1e-5 * float(ob.abs().max()), f"fp32 outputs differ by {err}"


class Run:
    """Drives a shared context and its twin with the same inputs."""

    def __init__(self, sh, tw, model, seed):
        self.sh, self.tw, self.model = sh, tw, model
        self.B = sh.B
        self.g = torch.Generator().manual_seed(seed)
        self.same = {}   # dst -> src: requests fed the same inputs
        self.lists = True   # compare the codes and the index lists too (they need save_mask)
        self.wins = None    # host copies of every request's window (track_windows): the oracle check of single steps
        self.tw_off = None  # keys each twin request stores

    def track_windows(self, doc, ws, hf):
        """Check single-token steps against the oracle fed the twin's stored state and these window copies (until a
        multi-token step: its rewind / accept are not mirrored)."""
        self.doc, self.hf = doc, hf
        self.wins = [(doc.wk[:, :w].clone(), doc.wv[:, :w].clone()) for w in ws]

    def oracle_check(self, q, k, v):
        k_st, v_st, kn_st = (x.cpu() for x in self.tw.read_cache(1))
        avg = self.doc.avg.reshape(1, Hkv, 1, d)
        nz_tw = self.tw.last_probe()[0].cpu()
        for b in range(self.B):
            n = self.model.n + len(self.model.vis[b])   # the twin request stores the prompt and its own spilled keys
            kd = k_st[b, :, :n].contiguous()
            t = dict(B=1, Hq=Hq, Hkv=Hkv, d=d, K=K, L=L, n=n, M=M, hash_func=self.hf, kcodes=self.tw.hash_keys(kd.to(DEV)).cpu()[None],
                     key=kd[None], value=v_st[b, :, :n][None].contiguous(), key_norm=kn_st[b, :, :n][None].contiguous(), avg_k=avg)
            qb = q[b:b + 1, 0].cpu().reshape(1, Hq, 1, d)
            kb, vb = (x[b:b + 1, 0].cpu().reshape(1, Hkv, 1, d) for x in (k, v))
            _, nz_ref, _, o_exact = oracle_decode(t, qb, kb, vb, self.wins[b][0][None], self.wins[b][1][None], Hq // Hkv)
            rows = slice(b * Hq, (b + 1) * Hq)
            assert torch.equal(nz_tw[rows], nz_ref), f"request {b}: twin nnz != oracle"
            for ctx in (self.tw, self.sh):
                assert_1e3_f32(ctx.last_out_f32()[rows].cpu(), o_exact)
            self.wins[b] = (torch.cat([self.wins[b][0], (kb - avg)[0]], dim=1), torch.cat([self.wins[b][1], vb[0]], dim=1))

    def qkv(self, T=1):
        q = torch.randn((self.B, T, Hq, d), generator=self.g).bfloat16()
        k = torch.randn((self.B, T, Hkv, d), generator=self.g).bfloat16()
        v = torch.randn((self.B, T, Hkv, d), generator=self.g).bfloat16()
        for dst, src in self.same.items():
            q[dst], k[dst], v[dst] = q[src], k[src], v[src]
        return q.to(DEV), k.to(DEV), v.to(DEV)

    def single(self, host=False):
        q, k, v = self.qkv()
        for ctx in (self.sh, self.tw):
            ctx.plan()
            if host:
                o = torch.zeros((self.B, Hq * d), dtype=torch.bfloat16).pin_memory()
                ctx.decode_host(1, q[:, 0].cpu().contiguous().pin_memory(), k[:, 0].cpu().contiguous().pin_memory(),
                                v[:, 0].cpu().contiguous().pin_memory(), o)
            else:
                ctx.decode(1, q[:, 0], k[:, 0], v[:, 0])
        compare(self.sh, self.tw, self.model, self.lists)
        if self.wins is not None:
            self.oracle_check(q, k, v)

    def tokens(self, drop):
        self.wins = None
        q, k, v = self.qkv(4)
        for ctx in (self.sh, self.tw):
            ctx.plan(4)
            ctx.decode_tokens(1, 4, q, k, v)
        compare(self.sh, self.tw, self.model, self.lists)
        dr = torch.tensor(drop, dtype=torch.int32, device=DEV)
        for ctx in (self.sh, self.tw):
            ctx.rewind(dr)

    def tree(self, nodes, count):
        self.wins = None
        par = torch.tensor([[-1, 0, 0, 1]] * self.B, dtype=torch.int32, device=DEV)
        q, k, v = self.qkv(4)
        for ctx in (self.sh, self.tw):
            ctx.plan(4, parents=par)
            ctx.decode_tokens(1, 4, q, k, v)
        compare(self.sh, self.tw, self.model, self.lists)
        nd = torch.tensor([nodes + [0] * (4 - len(nodes))] * self.B, dtype=torch.int32, device=DEV)
        ct = torch.tensor(count, dtype=torch.int32, device=DEV)
        for ctx in (self.sh, self.tw):
            ctx.accept(nd, ct)

    def spill(self, keep=NL):
        g = self.sh.spill_window(keep)
        assert g.tolist() == self.tw.spill_window(keep).tolist()
        self.model.spill(g.tolist())
        if self.wins is not None:
            for b, gb in enumerate(g.tolist()):
                self.wins[b] = tuple(torch.cat([w[:, :NS], w[:, NS + gb:]], dim=1) for w in self.wins[b])
        return g


def fill_windows(doc, ctxs, ws):
    for ctx in ctxs:
        for b, w in enumerate(ws):
            ctx.window_fill(1, b, doc.avg.to(DEV).contiguous(), doc.wk[:, :w].contiguous().to(DEV), doc.wv[:, :w].contiguous().to(DEV))


def seg_geometry(ctx):
    S = ctx.get_info("table_segments")
    return S, (((M + S - 1) // S) + 63) & ~63


VARIANTS = ["fused", "kreg", "cta512", "selcap", "nomask", "host", "three_launch"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_equivalence_to_exclusive_slots(cuda_lib, monkeypatch, variant):
    if variant == "cta512":
        monkeypatch.setenv("MPIG_CTA_PER_SM", "2")
    B = 3
    hf = synth.make_hash_func(d, K, L, seed=21)
    opts = dict(impl=0 if variant == "three_launch" else 1, kreg=1 if variant == "kreg" else 0,
                selcap=16 if variant == "selcap" else 2048, save_mask=0 if variant == "nomask" else 1)
    sh, tw = make_ctx(B, 1, hf, True, **opts), make_ctx(B, 0, hf, False, **opts)
    assert sh.get_info("shared_spill") == 1 and tw.get_info("shared_spill") == 0
    S, seg_len = seg_geometry(sh)
    if variant == "fused":
        assert S > 1, "the geometry no longer splits the private keys over key segments"
    # with several key segments the prompt ends 6 keys before a segment boundary: request 0's first 6 spilled keys fill the
    # prompt's last segment, the other requests' land in the next one
    n = seg_len - 6 if S > 1 else 1500
    doc = Doc(Hkv, n, K, L, hf, 700, w=NS + NL + 15)
    doc.fill_store(sh, 0)
    for b in range(B):
        doc.fill_store(tw, b)
    ws = [NS + NL + 3, NS + NL + 9, NS + NL + 15]
    fill_windows(doc, (sh, tw), ws)
    run = Run(sh, tw, Model(B, 1, n), seed=5)
    run.lists = variant != "nomask"
    if variant in ("fused", "three_launch"):   # both contexts against the oracle at every single step before the first T-token step
        run.track_windows(doc, ws, hf)
    multi = variant != "three_launch"
    for step in range(40):
        if step % 4 == 3:
            g = run.spill(NL if (step // 4) % 2 == 0 else NL - 16)
            if step == 3:
                assert g.tolist() == [6, 12, 18]
        if multi and step in (10, 22):
            run.tokens([0, 1, 3])
        elif multi and step in (17, 30):
            run.tree([0, 2], [2, 1, 0])
        else:
            run.single(host=variant == "host")
    assert sh.error_flags() == 0


def test_tables_fork_and_bind(cuda_lib):
    """B = 4 on two slots (0, 2 on slot 0; 1, 3 on slot 1), both filled with one document.  Requests 0 and 3 get the same inputs
    until 0 is forked to 3; then 2 is bound to slot 1 and refilled there."""
    B = 4
    hf = synth.make_hash_func(d, K, L, seed=31)
    sh, tw = make_ctx(B, 2, hf, True), make_ctx(B, 0, hf, False)
    n = 1500
    doc = Doc(Hkv, n, K, L, hf, 800, w=NS + NL + 12)
    doc.fill_store(sh, 0)
    doc.fill_store(sh, 1)
    for b in range(B):
        doc.fill_store(tw, b)
    ws = [NS + NL + 3, NS + NL + 8, NS + NL + 12, NS + NL + 3]
    fill_windows(doc, (sh, tw), ws)
    model = Model(B, 2, n)
    run = Run(sh, tw, model, seed=9)
    run.same = {3: 0}
    for _ in range(3):
        run.single()
    g = run.spill()
    assert g[0] > 0 and g[2] > 0
    # the tables of slot 0, into which requests 0 and 2 spilled, equal a device rebuild over every key the slot stores
    k_st = sh.read_cache(1, True, False, False)[0]
    ref = make_ctx(B, 2, hf, False)   # the same batch shape: the same key segments
    ref.lsh_build(1, 0, sh.hash_keys(k_st[0, :, : n + model.count[0]].contiguous()))
    o, i = lsh_tables(sh, 1)
    ro, ri = lsh_tables(ref, 1)
    assert_tables_equal((o[0], i[0]), (ro[0], ri[0]))
    for _ in range(3):
        run.single()
    run.spill(NL - 10)
    run.single()
    # fork 0 -> 3: request 3 (slot 1, its own spilled keys) moves to slot 0 and sees exactly request 0's spilled keys, whose
    # content equals that of the keys its twin spilled
    sh.fork(0, 3)
    model.fork(0, 3)
    run.same = {}
    for step in range(8):
        if step == 4:
            run.spill()
        run.single()
    # bind 2 -> slot 1: it sees no private key of slot 1 (request 1's and request 3's dead ones); its twin is refilled likewise
    sh.bind(2, 1)
    model.bind(2, 1)
    doc.fill_store(tw, 2)
    for ctx in (sh, tw):
        ctx.window_fill(1, 2, doc.avg.to(DEV).contiguous(), doc.wk[:, : NS + NL].contiguous().to(DEV),
                        doc.wv[:, : NS + NL].contiguous().to(DEV))
    for step in range(10):
        if step == 5:
            run.spill()
        run.single()
    run.tokens([1, 0, 2, 3])
    assert sh.error_flags() == 0


def test_graph_replays_across_spill_fork_bind(cuda_lib):
    hf = synth.make_hash_func(d, K, L, seed=41)
    doc = Doc(Hkv, 1500, K, L, hf, 900, w=NS + NL + 10)
    ctxs = []
    for _ in range(2):
        c = make_ctx(3, 1, hf, True)
        doc.fill_store(c, 0)
        fill_windows(doc, (c,), [NS + NL + 2, NS + NL + 6, NS + NL + 10])
        ctxs.append(c)
    g_ctx, e_ctx = ctxs
    q = torch.zeros((3, Hq, d), dtype=torch.bfloat16, device=DEV)
    k = torch.zeros((3, Hkv, d), dtype=torch.bfloat16, device=DEV)
    v = torch.zeros_like(k)
    out = torch.zeros((3, Hq * d), dtype=torch.bfloat16, device=DEV)
    for c in ctxs:
        c.plan()
        c.decode(1, q, k, v)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        g_ctx.plan()
        g_ctx.decode(1, q, k, v, out)
    gen = torch.Generator().manual_seed(6)

    def step():
        q.copy_(torch.randn((3, Hq, d), generator=gen).bfloat16())
        k.copy_(torch.randn((3, Hkv, d), generator=gen).bfloat16())
        v.copy_(torch.randn((3, Hkv, d), generator=gen).bfloat16())
        graph.replay()
        torch.cuda.synchronize()
        e_ctx.plan()
        ref = e_ctx.decode(1, q, k, v)
        assert torch.equal(out, ref)
        assert torch.equal(g_ctx.last_probe()[0], e_ctx.last_probe()[0])

    for _ in range(3):
        step()
    for c in ctxs:
        assert c.spill_window().sum() > 0
    for _ in range(3):
        step()
    for c in ctxs:
        c.fork(2, 0)
    for _ in range(2):
        step()
    for c in ctxs:
        c.bind(1, 0)
    for _ in range(2):
        step()


def test_refusals(cuda_lib):
    hf = synth.make_hash_func(d, 6, 24, seed=1)
    for B, C in ((3, 0), (3, 3), (33, 1)):
        with pytest.raises(N.MagicPigError, match="shared_spill"):
            Context(6, 24, 2, 4, 4, d, B, 400, NS, NL, GEN, dense_layers=[0], device=DEV, num_contexts=C, shared_spill=True)
    # a spill past max_length is refused and changes nothing: the next decode equals one of a context that never tried
    n, Mx = 1500, 1500 + 20
    hf_big = synth.make_hash_func(d, K, L, seed=2)
    ctxs = []
    for _ in range(2):
        c = Context(K, L, 2, Hq, Hkv, d, 2, Mx, NS, NL, GEN, dense_layers=[0], device=DEV, num_contexts=1, shared_spill=True)
        c.set_hash_func(hf_big.to(DEV))
        ctxs.append(c)
    doc = Doc(Hkv, n, K, L, hf_big, 50, w=NS + NL + 15)
    for c in ctxs:
        doc.fill_store(c, 0)
        for b in range(2):
            c.window_fill(1, b, doc.avg.to(DEV).contiguous(), doc.wk.contiguous().to(DEV), doc.wv.contiguous().to(DEV))
    a, b_ = ctxs
    before = lsh_tables(a, 1), a.read_cache(1)
    with pytest.raises(N.MagicPigError, match="max_length"):
        a.spill_window()   # 2 x 15 keys into 20 free rows
    after = lsh_tables(a, 1), a.read_cache(1)
    assert all(torch.equal(x, y) for x, y in zip(before[0], after[0]))
    assert all(torch.equal(x, y) for x, y in zip(before[1], after[1]))
    g = torch.Generator().manual_seed(3)
    q = torch.randn((2, Hq, d), generator=g).bfloat16().to(DEV)
    kv = torch.randn((2, Hkv, d), generator=g).bfloat16().to(DEV)
    outs = []
    for c in ctxs:
        c.plan()
        outs.append(c.decode(1, q, kv, kv).clone())
    assert torch.equal(outs[0], outs[1])
    # one request alone fits: its keys go in, and a refill of the slot leaves no request seeing them
    hf = synth.make_hash_func(d, K, L, seed=61)
    sh, tw = make_ctx(3, 1, hf, True), make_ctx(3, 0, hf, False)
    doc = Doc(Hkv, 1500, K, L, hf, 60, w=NS + NL + 10)
    doc.fill_store(sh, 0)
    for b in range(3):
        doc.fill_store(tw, b)
    fill_windows(doc, (sh, tw), [NS + NL + 4, NS + NL + 7, NS + NL + 10])
    model = Model(3, 1, 1500)
    run = Run(sh, tw, model, seed=4)
    run.single()
    run.spill()
    run.single()
    doc.fill_store(sh, 1)   # a refill through request 1 refills slot 0 for everybody
    for b in range(3):
        doc.fill_store(tw, b)
    model.refill(0)
    for _ in range(3):
        run.single()


def test_dropin_and_runner(cuda_lib):
    from magicpig_b200.attnserver import LSHSparseAttnServer
    cfg = _Cfg()
    cfg.num_hidden_layers, cfg.num_key_value_heads, cfg.num_attention_heads, cfg.hidden_size = 3, 2, 8, 8 * d
    B, P, gen_buf = 4, 1200, 16
    hf = torch.randn((d, 8 * 60), generator=torch.Generator().manual_seed(2)).bfloat16()
    mk = lambda C, s: LSHSparseAttnServer(cfg, K=8, L=60, batch_size=B, max_length=2048, dense_layers=(0,), device=DEV,  # noqa: E731
                                          hash_func=hf, generation_buffer=gen_buf, num_contexts=C, shared_spill=s)
    sh, tw = mk(1, True), mk(None, False)
    g = torch.Generator().manual_seed(3)
    kv = [(torch.randn((P, 2, d), generator=g).bfloat16().to(DEV), torch.randn((P, 2, d), generator=g).bfloat16().to(DEV)) for _ in range(3)]
    for srv, reqs in ((sh, [0]), (tw, range(B))):
        srv.alloc_buffer(P)
        for layer in range(3):
            for b in reqs:
                srv.fill(layer, b, kv[layer][0], kv[layer][1], P)
                srv.build_table(layer, b, P)
    sh.fork(0, [1, 2, 3])
    for step in range(3 * gen_buf):
        if step % 10 == 9:
            assert sh.spill_window().tolist() == tw.spill_window().tolist()
        q = torch.randn((B, 8, 1, d), generator=g).bfloat16().to(DEV)
        k = torch.randn((B, 2, 1, d), generator=g).bfloat16().to(DEV)
        for srv in (sh, tw):
            srv.plan()
        for layer in range(3):
            a, b_ = sh.decode(q, k, k, layer).float(), tw.decode(q, k, k, layer).float()
            assert float((a - b_).abs().max()) <= 1e-2 * float(b_.abs().max())
    assert sh.ctx.error_flags() == 0

    from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner
    runs = []
    for C, s in ((1, True), (None, False)):
        r = LlamaDecodeRunner(LLAMA31_8B, 8, 60, B, 4096, device=DEV, num_layers=3, num_contexts=C, generation_buffer=gen_buf,
                              shared_spill=s)
        r.synthetic_prefill(3000, shared=True)
        r.ids.copy_(torch.tensor([[11], [22], [33], [44]], device=DEV))
        r.capture()
        runs.append(r)
    for step in range(3 * gen_buf):
        if step % 10 == 9:
            for r in runs:
                r.server.spill_window()
        a, b_ = runs[0].replay().clone(), runs[1].replay().clone()
        torch.cuda.synchronize()
        if step < 3:
            assert float((a.float() - b_.float()).abs().max()) <= 0.25
            assert torch.equal(a.float().argmax(-1), b_.float().argmax(-1))
        assert torch.isfinite(a.float()).all()
    for r in runs:
        assert r.server.ctx.error_flags() == 0


def test_partial_refill_refused(cuda_lib):
    """Two sparse layers: after a spill, a refill of one of them leaves the slot's layers with different private key counts, and
    the next spill is refused with nothing changed (the next decode equals that of a context that never tried)."""
    hf = synth.make_hash_func(d, K, L, seed=71)
    doc = Doc(Hkv, 1500, K, L, hf, 90, w=NS + NL + 10)
    ctxs = []
    for _ in range(2):
        c = Context(K, L, 3, Hq, Hkv, d, 2, M, NS, NL, GEN, dense_layers=[0], device=DEV, num_contexts=1, shared_spill=True)
        c.set_hash_func(hf.to(DEV))
        kd = doc.key.to(DEV).contiguous()
        for layer in (1, 2):
            c.attn_fill(layer, 0, kd, doc.value.to(DEV).contiguous(), doc.kn.to(DEV).contiguous())
            c.lsh_build(layer, 0, doc.kcodes.to(DEV).contiguous())
            for b in range(2):
                c.window_fill(layer, b, doc.avg.to(DEV).contiguous(), doc.wk.contiguous().to(DEV), doc.wv.contiguous().to(DEV))
        ctxs.append(c)
    g = torch.Generator().manual_seed(8)

    def step():
        q = torch.randn((2, Hq, d), generator=g).bfloat16().to(DEV)
        kv = torch.randn((2, Hkv, d), generator=g).bfloat16().to(DEV)
        outs = []
        for c in ctxs:
            c.plan()
            outs.append([c.decode(layer, q, kv, kv).clone() for layer in (1, 2)])
        return outs

    step()
    for c in ctxs:
        assert c.spill_window().tolist() == [11, 11]
        doc.fill_store(c, 0)   # refills layer 1 only: layer 2 keeps its 22 private keys
    step()
    a = ctxs[0]
    before = [lsh_tables(a, layer) for layer in (1, 2)], [a.read_cache(layer) for layer in (1, 2)]
    with pytest.raises(N.MagicPigError, match="private keys"):
        a.spill_window()
    after = [lsh_tables(a, layer) for layer in (1, 2)], [a.read_cache(layer) for layer in (1, 2)]
    for x, y in zip(before, after):
        for tx, ty in zip(x, y):
            assert all(torch.equal(p, q_) for p, q_ in zip(tx, ty))
    outs = step()
    for layer in range(2):
        assert torch.equal(outs[0][layer], outs[1][layer])
