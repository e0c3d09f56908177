"""Compaction of a shared context (`-m gpu`): compact() drops the spilled keys no request sees any more and every request samples
exactly what it sampled before, up to the renumbering of the live keys.

The reference is the twin of test_gpu_shared_spill: every request owns its slot, filled with the same document and given the same
inputs and spills.  A host model keeps, per request, the private offsets it sees in the shared slot; compaction renumbers them
(live keys in time order to offsets 0, 1, ...).  A request must then match its twin: equal codes and nnz, equal index lists once
the shared slot's keys are mapped to the twin's, fp32 outputs within 1e-5 of the twin's largest output.  A beam reorder has no
exclusive twin, so there a shared context that never compacts is the reference, its keys mapped through the compaction.
"""
import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200 import synth
from magicpig_b200.ops import Context
from tests.support.fp64 import BAR, causal_ref, centred, rel_rows
from tests.support.library import DEV, NL, NS, Doc, assert_tables_equal, d, lsh_tables, two_layer_context

pytestmark = pytest.mark.gpu
GEN = 32
Hq, Hkv, K, L, M = 8, 2, 8, 60, 4096


def make_ctx(B, C, hf, shared, impl=1, kreg=0, save_mask=1, M_=M):
    return two_layer_context(K, L, Hq, Hkv, B, M_, GEN, hf, dict(decode_impl=impl, fused_kreg=kreg, out_f32=1, save_mask=save_mask),
                             max_query_tokens=4, num_contexts=C, shared_spill=shared)


def seg_len_of(ctx):
    S = ctx.get_info("table_segments")
    return S, (((ctx.M + S - 1) // S) + 63) & ~63


class Model:
    """Per slot the private offsets handed out so far, per request its slot and the offsets it sees (ascending)."""

    def __init__(self, B, C, n):
        self.n, self.slot = n, [b % C for b in range(B)]
        self.count = [0] * C
        self.vis = [[] for _ in range(B)]

    def spill(self, g):
        for b, gb in enumerate(g):
            c = self.slot[b]
            self.vis[b] += range(self.count[c], self.count[c] + gb)
            self.count[c] += gb

    def fork(self, src, dst):
        self.slot[dst], self.vis[dst] = self.slot[src], list(self.vis[src])

    def bind(self, r, c):
        self.slot[r], self.vis[r] = c, []

    def live(self, c):
        return sorted({p for b, v in enumerate(self.vis) if self.slot[b] == c for p in v})

    def compact(self, c):
        live = self.live(c)
        new = {p: j for j, p in enumerate(live)}
        for b in range(len(self.slot)):
            if self.slot[b] == c:
                self.vis[b] = [new[p] for p in self.vis[b]]
        dead = self.count[c] - len(live)
        self.count[c] = len(live)
        return dead

    def key_map(self, b):
        """shared slot key -> twin key for request b (-1: a key b must not see)"""
        mp = torch.full((M,), -1, dtype=torch.long, device=DEV)
        mp[: self.n] = torch.arange(self.n, device=DEV)
        if self.vis[b]:
            mp[self.n + torch.tensor(self.vis[b], device=DEV)] = self.n + torch.arange(len(self.vis[b]), device=DEV)
        return mp


def compare(sh, tw, maps, lists=True):
    """maps[b]: shared key -> reference key of request b"""
    B = sh.B
    nz_s, res_s = sh.last_probe(lists)
    nz_t, res_t = tw.last_probe(lists)
    assert torch.equal(nz_s, nz_t), "nnz differ"
    if lists:
        if sh.get_info("last_decode_fused"):
            assert torch.equal(sh.last_codes(), tw.last_codes()), "codes differ"
        per = nz_s.shape[0] // B
        valid = torch.arange(sh.M, device=DEV)[None] < nz_s[:, None]
        for b in range(B):
            r = slice(b * per, (b + 1) * per)
            mapped = maps[b][res_s[r].clamp(0, sh.M - 1).long()]
            assert bool((mapped[valid[r]] >= 0).all()), f"request {b} sampled a private key it does not see"
            assert torch.equal(torch.where(valid[r], mapped, -1), torch.where(valid[r], res_t[r].long(), -1)), f"request {b}: lists differ"
    oa, ob = sh.last_out_f32(), tw.last_out_f32()
    err = float((oa - ob).abs().max())
    assert err <= 1e-5 * float(ob.abs().max()), f"fp32 outputs differ by {err}"


class Run:
    """Drives a shared context and a reference with the same inputs; maps() gives each request's key map."""

    def __init__(self, sh, ref, maps, seed, lists=True):
        self.sh, self.ref, self.maps = sh, ref, maps
        self.B = sh.B
        self.g = torch.Generator().manual_seed(seed)
        self.same = {}
        self.lists = lists

    def qkv(self, T=1):
        q = torch.randn((self.B, T, Hq, d), generator=self.g).bfloat16()
        k = torch.randn((self.B, T, Hkv, d), generator=self.g).bfloat16()
        v = torch.randn((self.B, T, Hkv, d), generator=self.g).bfloat16()
        for dst, src in self.same.items():
            q[dst], k[dst], v[dst] = q[src], k[src], v[src]
        return q.to(DEV), k.to(DEV), v.to(DEV)

    def single(self, host=False):
        q, k, v = self.qkv()
        for ctx in (self.sh, self.ref):
            ctx.plan()
            if host:
                o = torch.zeros((self.B, Hq * d), dtype=torch.bfloat16).pin_memory()
                ctx.decode_host(1, q[:, 0].cpu().contiguous().pin_memory(), k[:, 0].cpu().contiguous().pin_memory(),
                                v[:, 0].cpu().contiguous().pin_memory(), o)
            else:
                ctx.decode(1, q[:, 0], k[:, 0], v[:, 0])
        compare(self.sh, self.ref, self.maps(), self.lists)

    def tokens(self, drop):
        q, k, v = self.qkv(4)
        for ctx in (self.sh, self.ref):
            ctx.plan(4)
            ctx.decode_tokens(1, 4, q, k, v)
        compare(self.sh, self.ref, self.maps(), self.lists)
        dr = torch.tensor(drop, dtype=torch.int32, device=DEV)
        for ctx in (self.sh, self.ref):
            ctx.rewind(dr)

    def tree(self, nodes, count):
        par = torch.tensor([[-1, 0, 0, 1]] * self.B, dtype=torch.int32, device=DEV)
        q, k, v = self.qkv(4)
        for ctx in (self.sh, self.ref):
            ctx.plan(4, parents=par)
            ctx.decode_tokens(1, 4, q, k, v)
        compare(self.sh, self.ref, self.maps(), self.lists)
        nd = torch.tensor([nodes + [0] * (4 - len(nodes))] * self.B, dtype=torch.int32, device=DEV)
        ct = torch.tensor(count, dtype=torch.int32, device=DEV)
        for ctx in (self.sh, self.ref):
            ctx.accept(nd, ct)

    def spill(self, keep=NL):
        g = self.sh.spill_window(keep)
        assert g.tolist() == self.ref.spill_window(keep).tolist()
        return g


def fill_windows(doc, ctxs, ws, reqs=None):
    for ctx in ctxs:
        for b, w in enumerate(ws):
            if reqs is None or b in reqs:
                ctx.window_fill(1, b, doc.avg.to(DEV).contiguous(), doc.wk[:, :w].contiguous().to(DEV), doc.wv[:, :w].contiguous().to(DEV))


def snapshot(ctx):
    return lsh_tables(ctx, 1), ctx.read_cache(1), ctx.visibility()


def same_state(a, b):
    (oa, ia), ca, va = a
    (ob, ib), cb, vb = b
    return torch.equal(oa, ob) and torch.equal(ia, ib) and all(torch.equal(x, y) for x, y in zip(ca, cb)) and torch.equal(va, vb)


def check_compaction(sh, hf, model, c, before, reclaimed):
    """State of slot c after compact(): the records, norms and vis words of the live keys moved down in order, zeros past the
    count, the tables a build over the compacted keys would make, and the count the host model expects."""
    n = model.n
    live = model.live(c)   # before the model's compaction: the old offsets, ascending
    dead = model.compact(c)
    assert reclaimed == dead
    (k0, v0, kn0), vis0 = before[1], before[2]
    k1, v1, kn1 = sh.read_cache(1)
    vis1 = sh.visibility()
    idx = torch.tensor(live, dtype=torch.long, device=DEV)
    j = len(live)
    for x0, x1 in ((k0, k1), (v0, v1), (kn0, kn1)):
        assert torch.equal(x1[c, :, n:n + j], x0[c, :, n + idx]), "live records moved wrongly"
        assert torch.equal(x1[c, :, :n], x0[c, :, :n]), "prompt records changed"
    assert torch.equal(vis1[c, :j], vis0[c, idx]) and bool((vis1[c, j:] == 0).all()), "vis not compacted"
    ref = make_ctx(sh.B, sh.C, hf, False)
    ref.lsh_build(1, 0, sh.hash_keys(k1[c, :, :n + j].contiguous()))
    o, i = lsh_tables(sh, 1)
    ro, ri = lsh_tables(ref, 1)
    assert_tables_equal((o[c], i[c]), (ro[0], ri[0]))


VARIANTS = ["fused", "kreg", "cta512", "host", "three_launch"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_equivalence_to_exclusive_slots(cuda_lib, monkeypatch, variant):
    """B = 3 on one slot whose prompt ends 6 keys below a key segment boundary.  Request 2 gets request 0's inputs, so its twin
    holds what request 0's holds.  Request 1 spills first, into both segments; then request 0's keys land in the upper segment.
    fork 0 -> 2 kills request 2's keys and a bind of 1 to the slot kills request 1's; compact() then moves request 0's live keys
    from the upper segment into the lower one.  More single-token steps, spills, T-token steps with rewind and trees follow."""
    if variant == "cta512":
        monkeypatch.setenv("MPIG_CTA_PER_SM", "2")
    B = 3
    hf = synth.make_hash_func(d, K, L, seed=21)
    opts = dict(impl=0 if variant == "three_launch" else 1, kreg=1 if variant == "kreg" else 0)
    sh, tw = make_ctx(B, 1, hf, True, **opts), make_ctx(B, 0, hf, False, **opts)
    S, seg_len = seg_len_of(sh)
    assert S > 1, "the geometry no longer splits the private keys over key segments"
    n = seg_len - 6
    doc = Doc(Hkv, n, K, L, hf, 700, w=NS + NL + 15)
    doc.fill_store(sh, 0)
    for b in range(B):
        doc.fill_store(tw, b)
    fill_windows(doc, (sh, tw), [NS + NL - 3, NS + NL + 9, NS + NL - 3])
    model = Model(B, 1, n)
    run = Run(sh, tw, lambda: [model.key_map(b) for b in range(B)], seed=5)
    run.same = {2: 0}
    multi = variant != "three_launch"
    host = variant == "host"

    def spill(keep=NL):
        g = run.spill(keep).tolist()
        model.spill(g)
        return g

    for step in range(8):
        if step % 4 == 3:
            g = spill()
            assert g == ([0, 12, 0] if step == 3 else [4, 4, 4])
        run.single(host)
    sh.fork(0, 2)   # the twin of 2 already holds what the twin of 0 holds
    model.fork(0, 2)
    sh.bind(1, 0)
    model.bind(1, 0)
    doc.fill_store(tw, 1)
    fill_windows(doc, (sh, tw), [NS + NL] * B, reqs=(1,))
    for _ in range(2):
        run.single(host)
    assert model.live(0) == [12, 13, 14, 15]
    before = snapshot(sh)
    reclaimed = sh.compact()
    assert reclaimed.shape == (1,) and int(reclaimed[0]) > 0
    check_compaction(sh, hf, model, 0, before, int(reclaimed[0]))
    # a second compaction has nothing to do and changes nothing
    again = snapshot(sh)
    assert sh.compact().tolist() == [0]
    assert same_state(again, snapshot(sh))
    assert tw.compact().tolist() == [0] * B   # no shared spill: nothing to reclaim
    run.same = {}
    for step in range(16):
        if step % 4 == 1:
            spill(NL if step % 8 == 1 else NL - 16)
        if multi and step == 6:
            run.tokens([0, 1, 3])
        elif multi and step == 10:
            run.tree([0, 2], [2, 1, 0])
        else:
            run.single(host)
    assert sh.error_flags() == 0



def test_two_slots_independently(cuda_lib):
    """B = 4 on two slots (0, 2 on slot 0; 1, 3 on slot 1).  Requests 2 and 3 mirror 0 and 1 until the forks 0 -> 2 and 1 -> 3
    kill their keys.  One compact() then reclaims both slots in one call (two slots' live keys staged, hashed and merged side by
    side); after more spills and the same forks, compact(0) reclaims slot 0 only and leaves slot 1's dead keys, tables and vis
    as they were, and compact(1) takes them.  Every request keeps matching its twin."""
    B = 4
    hf = synth.make_hash_func(d, K, L, seed=31)
    sh, tw = make_ctx(B, 2, hf, True), make_ctx(B, 0, hf, False)
    n = 1500
    doc = Doc(Hkv, n, K, L, hf, 800, w=NS + NL + 12)
    doc.fill_store(sh, 0)
    doc.fill_store(sh, 1)
    for b in range(B):
        doc.fill_store(tw, b)
    fill_windows(doc, (sh, tw), [NS + NL + 3, NS + NL + 8, NS + NL + 3, NS + NL + 8])
    model = Model(B, 2, n)
    run = Run(sh, tw, lambda: [model.key_map(b) for b in range(B)], seed=9)
    run.same = {2: 0, 3: 1}   # the twins of 2 and 3 hold what the twins of 0 and 1 hold

    def spill_and_fork():
        for step in range(8):
            if step % 4 == 3:
                model.spill(run.spill().tolist())
            run.single()
        for src, dst in ((0, 2), (1, 3)):
            sh.fork(src, dst)
            model.fork(src, dst)
        run.single()

    spill_and_fork()
    assert all(len(model.live(c)) < model.count[c] for c in (0, 1)) and all(model.live(c) for c in (0, 1))
    before = snapshot(sh)
    r = sh.compact()
    assert bool((r > 0).all()), r
    for c in (0, 1):
        check_compaction(sh, hf, model, c, before, int(r[c]))
    run.single()
    spill_and_fork()
    before = snapshot(sh)
    r0 = sh.compact(0)
    assert r0[0] > 0 and r0[1] == 0
    check_compaction(sh, hf, model, 0, before, int(r0[0]))
    after = snapshot(sh)
    assert torch.equal(before[0][0][1], after[0][0][1]) and torch.equal(before[0][1][1], after[0][1][1]), "slot 1's tables changed"
    assert all(torch.equal(x[1], y[1]) for x, y in zip(before[1], after[1])), "slot 1's store changed"
    assert torch.equal(before[2][1], after[2][1]), "slot 1's vis changed"
    r1 = sh.compact(1)
    assert r1[0] == 0 and r1[1] > 0
    check_compaction(sh, hf, model, 1, after, int(r1[1]))
    run.same = {}
    for step in range(8):
        if step == 4:
            model.spill(run.spill().tolist())
        run.single()
    run.tokens([1, 0, 2, 3])
    assert sh.error_flags() == 0


def test_chunk_step_after_compaction_vs_fp64(cuda_lib):
    """A chunk step reads the store length (store_n on the device, n_off on the host for its key splits) and vis, which the
    compaction rewrites.  Three requests on one slot spill 40 keys each; fork 1 -> 0 kills request 0's keys, the lowest ones, so
    the live keys of requests 1 and 2 move down.  A chunk of 64 tokens on the sparse layer is then held against fp64 at the 1e-3
    bar per request, each seeing the prompt and its own spilled keys; then the chunk is rewound, every request generates and
    spills again behind the compacted keys, and a second chunk is held to fp64 too."""
    B, Hq_, Hkv_, K_, L_, T = 3, 32, 8, 6, 16, 64
    G = Hq_ // Hkv_
    ctx = two_layer_context(K_, L_, Hq_, Hkv_, B, M, 320, synth.make_hash_func(d, K_, L_, seed=51), dict(out_f32=1),
                            alloc_dense_kv=True, num_contexts=1, shared_spill=True)
    ctx.reserve_chunk_tokens(T)
    g = torch.Generator(device=DEV).manual_seed(52)
    rnd = lambda *shape: torch.randn(shape, generator=g, device=DEV).bfloat16()   # noqa: E731
    n, p = 1337, 900
    sk, sv = rnd(Hkv_, n, d), rnd(Hkv_, n, d)
    ctx.attn_fill(1, 0, sk, sv, sk.float().norm(dim=-1).contiguous())
    ctx.lsh_build(1, 0, ctx.hash_keys(sk))
    ctx.dense_fill(0, 0, rnd(p, Hkv_, d), rnd(p, Hkv_, d), p)
    for b in range(1, B):
        ctx.fork(0, b)
    avg = [rnd(Hkv_, d) * 0.1 for _ in range(B)]
    wk = [rnd(Hkv_, NS + NL, d) for _ in range(B)]
    wv = [rnd(Hkv_, NS + NL, d) for _ in range(B)]
    for b in range(B):
        ctx.window_fill(1, b, avg[b].contiguous(), wk[b], wv[b])
    priv = [(wk[b][:, :0], wv[b][:, :0]) for b in range(B)]   # the spilled keys each request sees, in time order

    def generate(steps):
        for _ in range(steps):
            q, k, v = rnd(B, Hq_, 1, d), rnd(B, Hkv_, 1, d), rnd(B, Hkv_, 1, d)
            ctx.plan()
            ctx.decode(1, q, k, v)
            for b in range(B):
                wk[b] = torch.cat([wk[b], centred(k[b], avg[b][:, None])], 1)
                wv[b] = torch.cat([wv[b], v[b]], 1)

    def spill(steps):
        assert ctx.spill_window().tolist() == [steps] * B
        for b in range(B):
            priv[b] = (torch.cat([priv[b][0], wk[b][:, NS:NS + steps]], 1), torch.cat([priv[b][1], wv[b][:, NS:NS + steps]], 1))
            wk[b] = torch.cat([wk[b][:, :NS], wk[b][:, NS + steps:]], 1)
            wv[b] = torch.cat([wv[b][:, :NS], wv[b][:, NS + steps:]], 1)

    def chunk_vs_fp64(what):
        ctx.plan_chunk(T)
        q, k, v = rnd(B, T, Hq_, d), rnd(B, T, Hkv_, d), rnd(B, T, Hkv_, d)
        ctx.chunk_attend(1, T, q, k, v)
        f = ctx.last_out_f32().reshape(B, T, Hq_, d)
        for b in range(B):
            for h in range(Hkv_):
                kctx = torch.cat([sk[h], priv[b][0][h], wk[b][h]], 0)
                vctx = torch.cat([sv[h], priv[b][1][h], wv[b][h]], 0)
                ref = causal_ref(q[b, :, h * G:(h + 1) * G], kctx, vctx, centred(k[b, :, h], avg[b][h]), v[b, :, h])
                err = rel_rows(f[b, :, h * G:(h + 1) * G], ref)
                assert err <= BAR, f"{what}: request {b} kv-head {h}: {err:.3g} of the row max"
        ctx.rewind(torch.full((B,), T, dtype=torch.int32, device=DEV))

    generate(40)
    spill(40)
    ctx.fork(1, 0)
    wk[0], wv[0], avg[0], priv[0] = wk[1].clone(), wv[1].clone(), avg[1], priv[1]
    assert ctx.compact().tolist() == [40]
    ks = ctx.read_cache(1)[0][0]
    assert torch.equal(ks[:, n:n + 40], priv[1][0]) and torch.equal(ks[:, n + 40:n + 80], priv[2][0]), "live keys not moved down"
    chunk_vs_fp64("chunk after compact()")
    generate(30)
    spill(30)
    ks = ctx.read_cache(1)[0][0]
    assert torch.equal(ks[:, n + 80:n + 110], priv[0][0][:, 40:]), "a spill after compact() does not append behind the live keys"
    chunk_vs_fp64("chunk after compact() and a spill")
    assert ctx.error_flags() == 0


def test_reorder_then_compact(cuda_lib):
    """A beam reorder kills the keys of the lineages it drops.  Reference: a shared context given the same calls that never
    compacts; after compact() its keys are mapped through the live list, and later spills append in both."""
    B = 4
    hf = synth.make_hash_func(d, K, L, seed=37)
    a, r = make_ctx(B, 1, hf, True), make_ctx(B, 1, hf, True)
    n = 1500
    doc = Doc(Hkv, n, K, L, hf, 810, w=NS + NL + 12)
    for ctx in (a, r):
        doc.fill_store(ctx, 0)
    fill_windows(doc, (a, r), [NS + NL + 3, NS + NL + 6, NS + NL + 9, NS + NL + 12])
    amap = []      # private offset of `a` -> private offset of `r`
    count_r = [0]

    def maps():
        mp = torch.full((M,), -1, dtype=torch.long, device=DEV)
        mp[:n] = torch.arange(n, device=DEV)
        if amap:
            mp[n:n + len(amap)] = n + torch.tensor(amap, device=DEV)
        return [mp] * B

    run = Run(a, r, maps, seed=13)

    def spill():
        g = int(run.spill().sum())
        amap.extend(range(count_r[0], count_r[0] + g))
        count_r[0] += g

    for step in range(8):
        if step % 4 == 3:
            spill()
        run.single()
    src_of = torch.tensor([0, 0, 2, 2], dtype=torch.int32, device=DEV)
    for ctx in (a, r):
        ctx.reorder(src_of)
    run.single()
    vis = a.visibility()[0, :len(amap)]
    live = torch.nonzero(vis).flatten().tolist()
    assert a.compact().tolist() == [len(amap) - len(live)] and len(live) < len(amap)
    amap[:] = [amap[p] for p in live]
    for step in range(10):
        if step % 4 == 1:
            spill()
        run.single()
    run.tree([0, 2], [2, 1, 0, 2])
    run.single()
    assert a.error_flags() == 0


def test_capacity(cuda_lib):
    """A spill refused for max_length changes nothing, and succeeds once compact() has reclaimed the dead keys."""
    B, n = 3, 1500
    Mx = n + 60
    hf = synth.make_hash_func(d, K, L, seed=43)
    sh = make_ctx(B, 1, hf, True, M_=Mx)
    doc = Doc(Hkv, n, K, L, hf, 820, w=NS + NL + 10)
    doc.fill_store(sh, 0)
    fill_windows(doc, (sh,), [NS + NL + 10] * B)
    assert sh.spill_window().tolist() == [10, 10, 10]
    sh.fork(0, 1)
    sh.fork(0, 2)
    g = torch.Generator().manual_seed(2)
    for _ in range(11):
        sh.plan()
        sh.decode(1, *(torch.randn((B, h, d), generator=g).bfloat16().to(DEV) for h in (Hq, Hkv, Hkv)))
    before = snapshot(sh)
    with pytest.raises(N.MagicPigError, match="max_length"):
        sh.spill_window()   # 3 x 11 keys into 30 free rows
    assert same_state(before, snapshot(sh))
    assert sh.compact().tolist() == [20]
    assert sh.spill_window().tolist() == [11, 11, 11]
    sh.plan()
    out = sh.decode(1, *(torch.randn((B, h, d), generator=g).bfloat16().to(DEV) for h in (Hq, Hkv, Hkv)))
    assert bool(torch.isfinite(out.float()).all()) and sh.error_flags() == 0


def test_graph_replays_across_compaction(cuda_lib):
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
        assert int(c.compact()[0]) > 0
    for _ in range(3):
        step()
    for c in ctxs:
        assert c.spill_window().sum() > 0
        c.bind(1, 0)
        assert int(c.compact()[0]) > 0
    for _ in range(3):
        step()


def test_refusals(cuda_lib):
    """A bad slot, and a partial refill of one sparse layer: refused with nothing changed."""
    hf = synth.make_hash_func(d, K, L, seed=71)
    doc = Doc(Hkv, 1500, K, L, hf, 90, w=NS + NL + 10)
    c = Context(K, L, 3, Hq, Hkv, d, 2, M, NS, NL, GEN, dense_layers=[0], device=DEV, num_contexts=1, shared_spill=True)
    c.set_hash_func(hf.to(DEV))
    kd = doc.key.to(DEV).contiguous()
    for layer in (1, 2):
        c.attn_fill(layer, 0, kd, doc.value.to(DEV).contiguous(), doc.kn.to(DEV).contiguous())
        c.lsh_build(layer, 0, doc.kcodes.to(DEV).contiguous())
        for b in range(2):
            c.window_fill(layer, b, doc.avg.to(DEV).contiguous(), doc.wk.contiguous().to(DEV), doc.wv.contiguous().to(DEV))
    g = torch.Generator().manual_seed(8)
    c.plan()
    for layer in (1, 2):
        c.decode(layer, *(torch.randn((2, h, d), generator=g).bfloat16().to(DEV) for h in (Hq, Hkv, Hkv)))
    assert c.spill_window().tolist() == [11, 11]
    c.bind(1, 0)   # request 1's keys die
    for slot in (1, -2):
        with pytest.raises(N.MagicPigError, match="slot"):
            c.compact(slot)
    doc.fill_store(c, 0)   # refills layer 1 only: layer 2 keeps its 22 private keys
    state = lambda: ([lsh_tables(c, layer) for layer in (1, 2)], [c.read_cache(layer) for layer in (1, 2)], c.visibility())  # noqa: E731
    before = state()
    with pytest.raises(N.MagicPigError, match="private keys"):
        c.compact()
    after = state()
    for x, y in zip(before[:2], after[:2]):
        for tx, ty in zip(x, y):
            assert all(torch.equal(p, q_) for p, q_ in zip(tx, ty))
    assert torch.equal(before[2], after[2])


def test_runner_beam_search(cuda_lib):
    """A width-4 beam search with a captured step() + beam_step and a spill every generation_buffer steps, over a max_length
    too small for every spilled token: without compaction the spill is refused, with a compaction after each spill the search
    runs past that point.  The first compaction has nothing to reclaim (no spilled key is older than one window); every later
    one reclaims the keys of the lineages the reorders dropped since."""
    from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner
    W, P, gen_buf = 4, 3000, 16
    Mx = P + 3 * W * gen_buf + 10   # room for three spills of every beam

    def run(compact):
        r = LlamaDecodeRunner(LLAMA31_8B, 8, 60, W, Mx, device=DEV, num_layers=3, num_contexts=1, generation_buffer=gen_buf,
                              shared_spill=True, dense_tail_rows=128)
        scores = torch.zeros(W, dtype=torch.float32, device=DEV)
        r.synthetic_prefill(P, shared=True)
        r.capture(beam_scores=scores)
        r.server.clear()
        r.synthetic_prefill(P, shared=True)
        r.ids.fill_(17)
        scores.copy_(torch.tensor([0.0] + [float("-inf")] * (W - 1)))
        reclaimed = []
        for step in range(6 * gen_buf):
            if step and step % gen_buf == 0:
                r.server.spill_window()
                if compact:
                    reclaimed.append(int(r.server.compact()[0]))
            r.replay()
        torch.cuda.synchronize()
        assert bool(torch.isfinite(scores).all())
        assert r.server.ctx.error_flags() == 0
        return reclaimed

    with pytest.raises(N.MagicPigError, match="max_length"):
        run(False)
    reclaimed = run(True)
    assert len(reclaimed) == 5 and reclaimed[0] == 0 and all(x > 0 for x in reclaimed[1:]), reclaimed
