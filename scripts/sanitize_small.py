"""Small end-to-end cases of every hot-path kernel for compute-sanitizer (memcheck / racecheck / synccheck / initcheck).

    compute-sanitizer --tool memcheck python scripts/sanitize_small.py

Sizes are tiny (the tools slow kernels down 10-100x) but cover: the stand-alone SimHash / probe (uint8 tags, several clusters
shapes, two key segments) / gather-attention kernels, the fused single-launch decode (cluster of 8, cluster of 4 over two
segments, one CTA per head with codes from the SimHash kernel, several selection passes), the three-launch decode, the dense
kernel, the tensor-core key hash, the table build, the window spill, verification steps of T tokens, token trees with an accept,
requests sharing one context slot, shared spill (several requests of one slot spill, a fork, single-token and T-token decodes), and
the device-side reorder of requests (`reorder`: the in-place copy between requests, eager, refused and captured), the compaction
of a shared context (`compact`: eager and between replays of a captured step, against a twin), chunk steps
(`chunk`: the chunk attention kernel on sparse and dense layers with one and several key splits, a partial m-block and a partial last
tile, shared spill with private keys, the shared dense prefix, a rewind and a captured step), prefill attention (`prefill`: G = 7,
partial m-blocks and a partial last key tile, eager and captured), and BASELINE's C4 and C5 per-rank
geometry (`configs`: K11 L300 over 4 segments in clusters of 4, Hq 8 / Hkv 1 over 8 segments in clusters of 8).  Results are
also checked against each other so a tool run doubles as a test.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicpig_b200 import synth  # noqa: E402
from magicpig_b200.ops import Context  # noqa: E402

dev = "cuda:0"
d = 128


def decode_case(B, Hq, Hkv, n, K, L, selcap=2048, seed=0, tol=1e-5):
    M = n + 160
    g = torch.Generator(device=dev).manual_seed(seed)
    hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
    q = torch.randn((B * Hq, d), generator=g, device=dev).bfloat16()
    outs = {}
    for impl in (0, 1):
        ctx = Context(K, L, 1, Hq, Hkv, d, B, M, generation_buffer=8, device=dev)
        ctx.set_option("decode_impl", impl)
        ctx.set_option("fused_selcap", selcap)
        ctx.set_option("save_mask", 1)
        ctx.set_option("out_f32", 1)
        ctx.set_hash_func(hf)
        g2 = torch.Generator(device=dev).manual_seed(seed + 1)
        for b in range(B):
            key = torch.randn((Hkv, n, d), generator=g2, device=dev).bfloat16()
            val = torch.randn((Hkv, n, d), generator=g2, device=dev).bfloat16()
            ctx.attn_fill(0, b, key, val, key.norm(p=2, dim=-1).float())
            ctx.lsh_build(0, b, ctx.hash_keys(key))
            ctx.window_fill(0, b, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=dev),
                            torch.randn((Hkv, 68, d), generator=g2, device=dev).bfloat16(),
                            torch.randn((Hkv, 68, d), generator=g2, device=dev).bfloat16())
        for step in range(2):
            kn = torch.randn((B * Hkv, d), generator=g2, device=dev).bfloat16()
            vn = torch.randn((B * Hkv, d), generator=g2, device=dev).bfloat16()
            ctx.plan()
            out = ctx.decode(0, q, kn, vn)
        nnz, res = ctx.last_probe(want_results=True)
        mask = ctx.lsh_get_mask()
        torch.cuda.synchronize()
        assert ctx.get_info("last_decode_fused") == impl
        outs[impl] = (ctx.last_out_f32().cpu(), nnz.cpu(), res.cpu(), mask.cpu())
        del ctx
    a, b_ = outs[0], outs[1]
    assert torch.equal(a[1], b_[1]), "nnz differs between the decode variants"
    assert torch.equal(a[3], b_[3]), "masks differ"
    for h in range(B * Hq):
        assert torch.equal(a[2][h, : a[1][h]], b_[2][h, : b_[1][h]])
    assert float((a[0] - b_[0]).abs().max()) <= tol * float(a[0].abs().max())
    print(f"decode B={B} Hq={Hq} Hkv={Hkv} n={n} K={K} L={L} selcap={selcap}: nnz/head {float(a[1].float().mean()):.1f} ok")


def stage_case():
    B, Hq, Hkv, n, K, L = 2, 8, 2, 1000, 6, 24
    M = n + 24
    g = torch.Generator(device=dev).manual_seed(3)
    ctx = Context(K, L, 1, Hq, Hkv, d, B, M, dense_layers=[], device=dev)
    hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
    ctx.set_hash_func(hf)
    ctx.set_option("save_mask", 1)
    for b in range(B):
        key = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
        val = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
        ctx.attn_fill(0, b, key, val, key.norm(p=2, dim=-1).float())
        codes = synth.hash_keys(key, hf, K, L)
        sc, si = codes.sort()
        ctx.lsh_fill(0, b, sc.contiguous(), si.int().contiguous())   # sorted route
        ctx.lsh_build(0, b, codes)                                    # counting-sort route
    q = torch.randn((B * Hq, d), generator=g, device=dev).bfloat16()
    codes, qn = ctx.simhash(q)
    res = torch.zeros((B * Hq, M), dtype=torch.int32, device=dev)
    nnz = torch.zeros((B * Hq,), dtype=torch.int32, device=dev)
    ctx.lsh_batch_retrieve(0, codes, res, nnz)
    ctx.lsh_get_mask()
    ctx.lsh_collision_counts(0, codes)
    out = torch.zeros((B * Hq, d), dtype=torch.bfloat16, device=dev)
    mve = torch.zeros((2, B * Hq), dtype=torch.float32, device=dev)
    for tma in (1, 0):
        ctx.set_option("attend_tma", tma)
        ctx.attention_wrapper(0, K, L, out, mve, q, qn, res, nnz)
    ctx.read_cache(0)
    torch.cuda.synchronize()
    print(f"stages: nnz/head {float(nnz.float().mean()):.1f} ok")


def dense_case():
    B, Hq, Hkv, P = 2, 8, 2, 700
    M = 1024
    g = torch.Generator(device=dev).manual_seed(4)
    ctx = Context(4, 8, 1, Hq, Hkv, d, B, M, dense_layers=[0], alloc_dense_kv=True, device=dev)
    for b in range(B):
        ctx.dense_fill(0, b, torch.randn((P, Hkv, d), generator=g, device=dev).bfloat16(), torch.randn((P, Hkv, d), generator=g, device=dev).bfloat16(), P)
    ctx.plan()
    for impl in (1, 0):
        ctx.set_option("dense_impl", impl)
        ctx.dense_decode(0, torch.randn((B * Hq, d), generator=g, device=dev).bfloat16(), torch.randn((B * Hkv, d), generator=g, device=dev).bfloat16(),
                         torch.randn((B * Hkv, d), generator=g, device=dev).bfloat16())
    torch.cuda.synchronize()
    print("dense ok")


def host_and_peer_case():
    """mpig_decode_host (mapped pinned block, per-head flags polled by the host) and the world-size-1 peer exchange (push / wait /
    one-launch all-reduce kernels, the fused decode's gather epilogue)."""
    import torch.distributed as dist
    from magicpig_b200.peer import PeerExchange
    B, Hq, Hkv, n, K, L = 1, 8, 2, 1500, 8, 40
    M = n + 160
    g = torch.Generator(device=dev).manual_seed(9)
    ctx = Context(K, L, 1, Hq, Hkv, d, B, M, generation_buffer=16, device=dev)
    ctx.set_hash_func(torch.randn((d, K * L), generator=g, device=dev).bfloat16())
    key = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    ctx.attn_fill(0, 0, key, torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16(), key.norm(p=2, dim=-1).float())
    ctx.lsh_build(0, 0, ctx.hash_keys(key))
    ctx.window_fill(0, 0, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=dev), torch.randn((Hkv, 68, d), generator=g, device=dev).bfloat16(),
                    torch.randn((Hkv, 68, d), generator=g, device=dev).bfloat16())
    q = torch.randn((Hq, d), generator=g, device=dev).bfloat16()
    kn, vn = torch.randn((Hkv, d), generator=g, device=dev).bfloat16(), torch.randn((Hkv, d), generator=g, device=dev).bfloat16()
    ctx.plan()
    ref = ctx.decode(0, q, kn, vn).clone()
    out_h = torch.zeros((B, Hq * d), dtype=torch.bfloat16).pin_memory()
    ctx.decode_host(0, q.cpu().pin_memory(), kn.cpu().pin_memory(), vn.cpu().pin_memory(), out_h)   # same window slot, same row
    assert torch.equal(out_h.to(dev), ref)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29533")
    dist.init_process_group("gloo", rank=0, world_size=1)
    px = PeerExchange(ctx, 0, 1, B * Hq * d * 2)
    for _ in range(3):
        a = torch.randn((B, Hq * d), generator=g, device=dev).bfloat16()
        assert torch.equal(px.all_gather(a), a)
        t = torch.randn((B, 512), generator=g, device=dev).bfloat16()
        t0 = t.clone()
        assert torch.equal(px.all_reduce(t), t0)
    assert torch.equal(px.decode_allgather(0, q, kn, vn), ref)
    torch.cuda.synchronize()
    px.close()
    dist.destroy_process_group()
    print("host buffers + peer exchange ok")


def spill_case():
    """Window spill (store move + norms, key hash of the spilled keys, table merge across a segment boundary) followed by a decode;
    the tables must equal a device rebuild over all stored keys."""
    B, Hq, Hkv, n, K, L, M = 1, 4, 2, 1000, 6, 16, 4096   # 4 segments of 1024 keys: the spill crosses 1024
    g = torch.Generator(device=dev).manual_seed(12)
    hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
    ctxs = []
    for _ in range(2):
        ctx = Context(K, L, 1, Hq, Hkv, d, B, M, generation_buffer=40, device=dev)
        ctx.set_hash_func(hf)
        ctxs.append(ctx)
    ctx, other = ctxs
    key = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    ctx.attn_fill(0, 0, key, torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16(), key.norm(p=2, dim=-1).float())
    ctx.lsh_build(0, 0, ctx.hash_keys(key))
    ctx.window_fill(0, 0, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=dev), torch.randn((Hkv, 68, d), generator=g, device=dev).bfloat16(),
                    torch.randn((Hkv, 68, d), generator=g, device=dev).bfloat16())
    q = torch.randn((B * Hq, d), generator=g, device=dev).bfloat16()
    for _ in range(40):
        ctx.plan()
        ctx.decode(0, q, torch.randn((B * Hkv, d), generator=g, device=dev).bfloat16(), torch.randn((B * Hkv, d), generator=g, device=dev).bfloat16())
    assert ctx.spill_window().tolist() == [40]
    ctx.plan()
    ctx.decode(0, q, torch.randn((B * Hkv, d), generator=g, device=dev).bfloat16(), torch.randn((B * Hkv, d), generator=g, device=dev).bfloat16())
    k_st, _, _ = ctx.read_cache(0, True, False, False)
    other.lsh_build(0, 0, ctx.hash_keys(k_st[0, :, : n + 40].contiguous()))
    torch.cuda.synchronize()
    from ctypes import byref, c_void_p

    class _View:   # a device buffer the library owns, seen by torch without a copy
        def __init__(self, ptr, count):
            self.__cuda_array_interface__ = {"shape": (count,), "typestr": "<i4", "data": (ptr, False), "version": 2}

    count = B * Hkv * L * ctx.get_info("table_segments") * ((1 << K) + 1)
    offs = []
    for c in (ctx, other):
        p = c_void_p()
        c.lib.mpig_lsh_table_ptrs(c._h, 0, byref(p), None)
        offs.append(torch.as_tensor(_View(p.value, count), device=dev))
    assert torch.equal(offs[0], offs[1]), "tables after the spill differ from a rebuild"
    print("spill ok")


def tokens_case(B, Hq, Hkv, n, K, L, T):
    """A verification step of T tokens (row append, the T-token fused kernel / SimHash kernel over B*T*Hq rows, the T-token dense
    kernel, rewind) against T single-token steps of a twin context."""
    M = n + 160
    g = torch.Generator(device=dev).manual_seed(20 + T)
    hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
    ctxs = []
    for tmax in (T, 1):
        ctx = Context(K, L, 2, Hq, Hkv, d, B, M, generation_buffer=16, dense_layers=[0], alloc_dense_kv=True, device=dev,
                      max_query_tokens=tmax)
        ctx.set_option("out_f32", 1)
        ctx.set_hash_func(hf)
        ctxs.append(ctx)
    g2 = torch.Generator(device=dev).manual_seed(21)
    for b in range(B):
        key = torch.randn((Hkv, n, d), generator=g2, device=dev).bfloat16()
        val = torch.randn((Hkv, n, d), generator=g2, device=dev).bfloat16()
        wk, wv = (torch.randn((Hkv, 68, d), generator=g2, device=dev).bfloat16() for _ in range(2))
        dk, dv = (torch.randn((300, Hkv, d), generator=g2, device=dev).bfloat16() for _ in range(2))
        for ctx in ctxs:
            ctx.attn_fill(1, b, key, val, key.norm(p=2, dim=-1).float())
            ctx.lsh_build(1, b, ctx.hash_keys(key))
            ctx.window_fill(1, b, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=dev), wk, wv)
            ctx.dense_fill(0, b, dk, dv, 300)
    q = torch.randn((B, T, Hq, d), generator=g, device=dev).bfloat16()
    k, v = (torch.randn((B, T, Hkv, d), generator=g, device=dev).bfloat16() for _ in range(2))
    tok, seq = ctxs
    tok.plan(T)
    tok.decode_tokens(1, T, q, k, v)
    o_s = tok.last_out_f32().reshape(B, T, Hq, d)
    tok.dense_decode_tokens(0, T, q, k, v)
    o_d = tok.last_out_f32().reshape(B, T, Hq, d)
    tok.rewind(torch.full((B,), 1, dtype=torch.int32, device=dev))
    for t in range(T):
        seq.plan()
        seq.decode(1, q[:, t].contiguous(), k[:, t].contiguous(), v[:, t].contiguous())
        r_s = seq.last_out_f32().reshape(B, Hq, d)
        seq.dense_decode(0, q[:, t].contiguous(), k[:, t].contiguous(), v[:, t].contiguous())
        r_d = seq.last_out_f32().reshape(B, Hq, d)
        for a, r in ((o_s[:, t], r_s), (o_d[:, t], r_d)):
            assert float((a - r).abs().max()) <= 1e-5 * float(r.abs().max()), f"token {t} differs from the single-token step"
    torch.cuda.synchronize()
    print(f"tokens B={B} Hq={Hq} Hkv={Hkv} n={n} T={T}: waves {tok.get_info('tokens_cluster_waves')} ok")


def tree_case(B, Hq, Hkv, n, K, L, parents, path):
    """A token-tree step (the plan kernel's ancestor masks, the masked T-token fused and dense kernels, the accept kernel moving
    rows in every layer): every node against a chain step over its root path on a twin context, then accept(path) on one and the
    path as a chain step on the other, and one more token on both."""
    T = len(parents)
    assert path[-1] == T - 1, "the twin keeps the accepted path's chain step, so it must be the last one it runs"
    M = n + 160
    g = torch.Generator(device=dev).manual_seed(30 + T)
    hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
    ctxs = []
    for _ in range(2):
        ctx = Context(K, L, 2, Hq, Hkv, d, B, M, generation_buffer=16, dense_layers=[0], alloc_dense_kv=True, device=dev,
                      max_query_tokens=T)
        ctx.set_option("out_f32", 1)
        ctx.set_hash_func(hf)
        ctxs.append(ctx)
    g2 = torch.Generator(device=dev).manual_seed(31)
    for b in range(B):
        key = torch.randn((Hkv, n, d), generator=g2, device=dev).bfloat16()
        val = torch.randn((Hkv, n, d), generator=g2, device=dev).bfloat16()
        wk, wv = (torch.randn((Hkv, 68, d), generator=g2, device=dev).bfloat16() for _ in range(2))
        dk, dv = (torch.randn((300, Hkv, d), generator=g2, device=dev).bfloat16() for _ in range(2))
        for ctx in ctxs:
            ctx.attn_fill(1, b, key, val, key.norm(p=2, dim=-1).float())
            ctx.lsh_build(1, b, ctx.hash_keys(key))
            ctx.window_fill(1, b, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=dev), wk, wv)
            ctx.dense_fill(0, b, dk, dv, 300)
    q = torch.randn((B, T, Hq, d), generator=g, device=dev).bfloat16()
    k, v = (torch.randn((B, T, Hkv, d), generator=g, device=dev).bfloat16() for _ in range(2))
    tree, ref = ctxs

    def root_path(t):
        p = [t]
        while parents[p[-1]] >= 0:
            p.append(parents[p[-1]])
        return p[::-1]

    tree.plan(T, parents=torch.tensor([parents] * B, dtype=torch.int32, device=dev))
    tree.decode_tokens(1, T, q, k, v)
    o_s = tree.last_out_f32().reshape(B, T, Hq, d).clone()
    tree.dense_decode_tokens(0, T, q, k, v)
    o_d = tree.last_out_f32().reshape(B, T, Hq, d).clone()
    tree.accept(torch.tensor([path + [0] * (T - len(path))] * B, dtype=torch.int32, device=dev),
                torch.full((B,), len(path), dtype=torch.int32, device=dev))
    for t in range(T):
        p = root_path(t)
        ref.plan(len(p))
        ref.decode_tokens(1, len(p), q[:, p].contiguous(), k[:, p].contiguous(), v[:, p].contiguous())
        r_s = ref.last_out_f32().reshape(B, len(p), Hq, d)[:, -1]
        ref.dense_decode_tokens(0, len(p), q[:, p].contiguous(), k[:, p].contiguous(), v[:, p].contiguous())
        r_d = ref.last_out_f32().reshape(B, len(p), Hq, d)[:, -1]
        ref.rewind(torch.full((B,), 0 if p == path else len(p), dtype=torch.int32, device=dev))
        for a, r in ((o_s[:, t], r_s), (o_d[:, t], r_d)):
            assert float((a - r).abs().max()) <= 1e-5 * float(r.abs().max()), f"node {t} differs from its path's chain step"
    q1 = torch.randn((B, 1, Hq, d), generator=g, device=dev).bfloat16()
    k1, v1 = (torch.randn((B, 1, Hkv, d), generator=g, device=dev).bfloat16() for _ in range(2))
    outs = []
    for ctx in ctxs:
        ctx.plan(1)
        outs.append(ctx.decode_tokens(1, 1, q1, k1, v1).clone())
        outs.append(ctx.dense_decode_tokens(0, 1, q1, k1, v1).clone())
    assert torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[3]), "state after accept differs from the path's chain"
    assert tree.error_flags() == 0
    torch.cuda.synchronize()
    print(f"tree B={B} Hq={Hq} Hkv={Hkv} n={n} T={T}: ok")


def shared_case(B, Hq, Hkv, n, K, L):
    """Context slots: request 0 filled and forked to the others over one slot (the fused kernel, the three-launch path's probe and
    gather kernels reading the slot map), a bind, and a refused spill; every decode against a twin that holds B copies."""
    M = n + 160
    g = torch.Generator(device=dev).manual_seed(40)
    hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
    ctxs = []
    for C in (1, 0):
        ctx = Context(K, L, 2, Hq, Hkv, d, B, M, generation_buffer=16, dense_layers=[0], alloc_dense_kv=True, device=dev,
                      num_contexts=C)
        ctx.set_option("out_f32", 1)
        ctx.set_hash_func(hf)
        ctxs.append(ctx)
    sh, tw = ctxs
    key = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    val = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    wk, wv = (torch.randn((Hkv, 68, d), generator=g, device=dev).bfloat16() for _ in range(2))
    dk, dv = (torch.randn((300, Hkv, d), generator=g, device=dev).bfloat16() for _ in range(2))
    for ctx, reqs in ((sh, [0]), (tw, range(B))):
        for b in reqs:
            ctx.attn_fill(1, b, key, val, key.norm(p=2, dim=-1).float())
            ctx.lsh_build(1, b, ctx.hash_keys(key))
            ctx.window_fill(1, b, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=dev), wk, wv)
            ctx.dense_fill(0, b, dk, dv, 300)
    for b in range(1, B):
        sh.fork(0, b)
    sh.bind(B - 1, 0)
    for impl in (1, 0):
        q = torch.randn((B * Hq, d), generator=g, device=dev).bfloat16()
        k, v = (torch.randn((B * Hkv, d), generator=g, device=dev).bfloat16() for _ in range(2))
        outs = []
        for ctx in ctxs:
            ctx.set_option("decode_impl", impl)
            ctx.plan()
            ctx.decode(1, q, k, v)
            outs.append(ctx.last_out_f32())
            ctx.dense_decode(0, q, k, v)
            outs.append(ctx.last_out_f32())
        assert float((outs[0] - outs[2]).abs().max()) <= 1e-5 and torch.equal(outs[1], outs[3]), f"impl {impl}: shared != twin"
    try:
        sh.spill_window(0)
        raise AssertionError("a spill into a shared slot was accepted")
    except Exception as e:   # refused: the requests share slot 0 and their windows are not empty
        assert "shares" in str(e), e
    torch.cuda.synchronize()
    print(f"shared B={B} Hq={Hq} Hkv={Hkv} n={n}: ok")


def shared_spill_case(B, Hq, Hkv, n, K, L, T):
    """B requests on one slot in shared spill mode against a twin with one slot per request: every request spills (the visibility
    writes of spill_move_kernel, the per-slot merge), single-token and T-token decodes (the filter of the fused and probe kernels),
    then a fork (vis_rebind_kernel) after which the forked request, fed the same inputs as its source, decodes exactly like it."""
    M = n + 400
    g = torch.Generator(device=dev).manual_seed(11)
    hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
    key = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    val = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    ctxs = []
    for C, shared in ((1, True), (0, False)):
        ctx = Context(K, L, 1, Hq, Hkv, d, B, M, num_local_tokens=64, generation_buffer=24, device=dev, max_query_tokens=T,
                      num_contexts=C, shared_spill=shared)
        ctx.set_option("save_mask", 1)
        ctx.set_option("out_f32", 1)
        ctx.set_hash_func(hf)
        for b in (range(1) if shared else range(B)):
            ctx.attn_fill(0, b, key, val, key.norm(p=2, dim=-1).float())
            ctx.lsh_build(0, b, ctx.hash_keys(key))
        g2 = torch.Generator(device=dev).manual_seed(12)
        for b in range(B):
            w = 68 + 4 * b   # different window lengths: different spill sizes
            ctx.window_fill(0, b, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=dev),
                            torch.randn((Hkv, w, d), generator=g2, device=dev).bfloat16(),
                            torch.randn((Hkv, w, d), generator=g2, device=dev).bfloat16())
        ctxs.append(ctx)
    sh, tw = ctxs
    for step in range(4):
        if step == 2:
            spilled = [c.spill_window(48).tolist() for c in ctxs]
            assert spilled[0] == spilled[1] and min(spilled[0]) > 0, spilled
        for impl in (1, 0):
            q = torch.randn((B * Hq, d), generator=g, device=dev).bfloat16()
            kv = torch.randn((B * Hkv, d), generator=g, device=dev).bfloat16()
            nz = []
            for c in ctxs:
                c.set_option("decode_impl", impl)
                c.plan()
                c.decode(0, q, kv, kv)
                nz.append((c.last_probe()[0], c.last_out_f32()))
            assert torch.equal(nz[0][0], nz[1][0]) and float((nz[0][1] - nz[1][1]).abs().max()) <= 1e-5 * float(nz[1][1].abs().max()), \
                f"step {step} impl {impl}: shared != twin"
    q = torch.randn((B, T, Hq, d), generator=g, device=dev).bfloat16()
    kv = torch.randn((B, T, Hkv, d), generator=g, device=dev).bfloat16()
    nz = []
    for c in ctxs:
        c.set_option("decode_impl", 1)
        c.plan(T)
        c.decode_tokens(0, T, q, kv, kv)
        nz.append(c.last_probe()[0])
        c.rewind(torch.zeros(B, dtype=torch.int32, device=dev))
    assert torch.equal(nz[0], nz[1]), "T-token step: shared != twin"
    sh.fork(0, B - 1)
    q = torch.randn((B, Hq, d), generator=g, device=dev).bfloat16()
    kv = torch.randn((B, Hkv, d), generator=g, device=dev).bfloat16()
    q[B - 1], kv[B - 1] = q[0], kv[0]
    sh.plan()
    sh.decode(0, q, kv, kv)
    nnz, res = sh.last_probe(want_results=True)
    o = sh.last_out_f32()
    torch.cuda.synchronize()
    a, b_ = slice(0, Hq), slice((B - 1) * Hq, B * Hq)
    valid = torch.arange(M, device=dev)[None] < nnz[a, None]
    assert torch.equal(nnz[a], nnz[b_]) and torch.equal(torch.where(valid, res[a], -1), torch.where(valid, res[b_], -1)) \
        and torch.equal(o[a], o[b_]), "fork: dst != src"
    print(f"shared spill B={B} Hq={Hq} Hkv={Hkv} n={n} T={T}: ok")


def compact_case(B, C, Hq, Hkv, n, K, L):
    """mpig_compact_context on C slots against a twin with one slot per request: request B-1-i is fed request i's inputs
    (i < C, request b starts on slot b % C), so a fork i -> B-1-i kills the private keys it left in its slot and leaves its twin
    right.  With C = 2 both slots then hold dead keys and one compact() reclaims both (their live keys staged, hashed and merged
    side by side).  compact() (the live list, the in-place record / vis move, the key staging, the table truncate and merge)
    runs eagerly and between two replays of a step captured before it; every decode matches the twin in nnz and within 1e-5 in
    fp32."""
    M = n + 400
    g = torch.Generator(device=dev).manual_seed(21)
    hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
    key = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    val = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    ctxs = []
    mirror = {B - 1 - i: i for i in range(C)}
    for nc, shared in ((C, True), (0, False)):
        ctx = Context(K, L, 1, Hq, Hkv, d, B, M, num_local_tokens=64, generation_buffer=24, device=dev, num_contexts=nc,
                      shared_spill=shared)
        ctx.set_option("out_f32", 1)
        ctx.set_hash_func(hf)
        for b in (range(C) if shared else range(B)):
            ctx.attn_fill(0, b, key, val, key.norm(p=2, dim=-1).float())
            ctx.lsh_build(0, b, ctx.hash_keys(key))
        g2 = torch.Generator(device=dev).manual_seed(22)
        wins = [(torch.randn((Hkv, 68 + 4 * b, d), generator=g2, device=dev).bfloat16(),
                 torch.randn((Hkv, 68 + 4 * b, d), generator=g2, device=dev).bfloat16()) for b in range(B)]
        for b in range(B):   # request B - 1 - i starts as a copy of request i
            ctx.window_fill(0, b, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=dev), *wins[mirror.get(b, b)])
        ctxs.append(ctx)
    sh, tw = ctxs
    q = torch.zeros((B * Hq, d), dtype=torch.bfloat16, device=dev)
    kv = torch.zeros((B * Hkv, d), dtype=torch.bfloat16, device=dev)
    out = torch.zeros((B, Hq * d), dtype=torch.bfloat16, device=dev)
    for c in ctxs:
        c.plan()
        c.decode(0, q, kv, kv)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        sh.plan()
        sh.decode(0, q, kv, kv, out)

    def step(replay):
        q.copy_(torch.randn((B * Hq, d), generator=g, device=dev).bfloat16())
        kv.copy_(torch.randn((B * Hkv, d), generator=g, device=dev).bfloat16())
        for dst, src in mirror.items():
            q.view(B, Hq, d)[dst], kv.view(B, Hkv, d)[dst] = q.view(B, Hq, d)[src], kv.view(B, Hkv, d)[src]
        if replay:
            graph.replay()
        else:
            sh.plan()
            sh.decode(0, q, kv, kv, out)
        tw.plan()
        tw.decode(0, q, kv, kv)
        torch.cuda.synchronize()
        o_s, o_t = sh.last_out_f32(), tw.last_out_f32()
        assert torch.equal(sh.last_probe()[0], tw.last_probe()[0]) and float((o_s - o_t).abs().max()) <= 1e-5 * float(o_t.abs().max()), \
            "compacted shared context != twin"

    for rnd in range(2):
        for c in ctxs:
            assert c.spill_window(48).sum() > 0
        step(False)
        for dst, src in mirror.items():
            sh.fork(src, dst)   # the twin of dst already holds what the twin of src holds
        reclaimed = sh.compact()
        assert bool((reclaimed > 0).all()), reclaimed
        step(rnd == 1)
        step(rnd == 1)
    print(f"compact B={B} C={C} Hq={Hq} Hkv={Hkv} n={n}: ok")


def reorder_case(B, Hq, Hkv, n, K, L, R):
    """mpig_reorder_requests: the in-place copy of windows, avg_k and dense tails between requests of one slot (shared dense mode,
    shared spill: the visibility rewrite of the same launch) and the slot-map staging, against a twin that forks request by request;
    then a bad map (nothing changes), and a reorder captured into a graph and replayed."""
    M = n + 400
    g = torch.Generator(device=dev).manual_seed(21)
    hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
    key = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    val = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    dk, dv = (torch.randn((300, Hkv, d), generator=g, device=dev).bfloat16() for _ in range(2))
    ctxs = []
    for _ in range(2):
        ctx = Context(K, L, 2, Hq, Hkv, d, B, M, generation_buffer=24, dense_layers=[0], alloc_dense_kv=True, device=dev,
                      num_contexts=2, dense_tail_rows=R, shared_spill=True)
        ctx.set_option("out_f32", 1)
        ctx.set_hash_func(hf)
        g2 = torch.Generator(device=dev).manual_seed(22)
        for c in range(2):
            ctx.attn_fill(1, c, key, val, key.norm(p=2, dim=-1).float())
            ctx.lsh_build(1, c, ctx.hash_keys(key))
        for b in range(B):
            ctx.window_fill(1, b, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=dev),
                            torch.randn((Hkv, 68, d), generator=g2, device=dev).bfloat16(),
                            torch.randn((Hkv, 68, d), generator=g2, device=dev).bfloat16())
            ctx.dense_fill(0, b, dk, dv, 300)
        ctxs.append(ctx)
    sh, tw = ctxs

    def step():
        q = torch.randn((B * Hq, d), generator=g, device=dev).bfloat16()
        kv = torch.randn((B * Hkv, d), generator=g, device=dev).bfloat16()
        outs = []
        for c in ctxs:
            c.plan()
            c.dense_decode(0, q, kv, kv)
            outs.append(c.last_out_f32())
            c.decode(1, q, kv, kv)
            outs.append(c.last_out_f32())
        assert torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[3]), "reorder != forks"

    def forks(m):
        for b, s_ in enumerate(m):
            if s_ != b:
                tw.fork(s_, b)

    for _ in range(3):
        step()
    assert sh.spill_window(64).tolist() == tw.spill_window(64).tolist()
    m = [0, 0, 2, 0][:B]
    sh.reorder(torch.tensor(m, dtype=torch.int32, device=dev))
    forks(m)
    step()
    try:
        sh.reorder(torch.tensor([1, 2, 2, 3][:B], dtype=torch.int32, device=dev))
        raise AssertionError("a map whose source is moved was accepted")
    except Exception as e:
        assert "code -1" in str(e), e
    step()
    src = torch.tensor([2, 1, 2, 2][:B], dtype=torch.int32, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            sh.reorder(src)
    torch.cuda.synchronize()
    graph.replay()
    forks(src.tolist())
    step()
    assert sh.error_flags() == 16 and tw.error_flags() == 0
    torch.cuda.synchronize()
    print(f"reorder B={B} Hq={Hq} Hkv={Hkv} n={n} R={R}: ok")


def chunk_case(B, Hq, Hkv, n, K, L, T, R):
    """Chunk steps: B requests on one slot (shared spill, dense prefix with R tail rows) against a twin with one slot per request and
    a full dense cache each.  Both get the same prompt, windows and 30 generated tokens on both layers, spill (private keys in the
    shared slot), then a chunk of T on the sparse layer 1 and the dense layer 0 (T*G rows: a partial second m-block when T*G > 128;
    n decides one key split or several), a rewind of part of it, a second chunk, and that second chunk captured into a graph and
    replayed.  Shared and twin agree to summation order; the replay equals the eager call."""
    M = n + 600
    g = torch.Generator(device=dev).manual_seed(21)
    hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
    key = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    val = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    dk = torch.randn((n, Hkv, d), generator=g, device=dev).bfloat16()
    ctxs = []
    for shared in (True, False):
        ctx = Context(K, L, 2, Hq, Hkv, d, B, M, num_local_tokens=64, generation_buffer=T + 40, dense_layers=[0], alloc_dense_kv=True,
                      device=dev, num_contexts=1 if shared else 0, dense_tail_rows=R if shared else 0, shared_spill=shared)
        ctx.set_option("out_f32", 1)
        ctx.set_hash_func(hf)
        ctx.reserve_chunk_tokens(T)
        for b in (range(1) if shared else range(B)):
            ctx.attn_fill(1, b, key, val, key.norm(p=2, dim=-1).float())
            ctx.lsh_build(1, b, ctx.hash_keys(key))
            ctx.dense_fill(0, b, dk, dk, n)
        for b in range(1, B if shared else 1):
            ctx.fork(0, b)
        g2 = torch.Generator(device=dev).manual_seed(22)
        for b in range(B):
            w = 68 + 5 * b
            ctx.window_fill(1, b, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=dev),
                            torch.randn((Hkv, w, d), generator=g2, device=dev).bfloat16(),
                            torch.randn((Hkv, w, d), generator=g2, device=dev).bfloat16())
        ctxs.append(ctx)
    for _ in range(30):
        q = torch.randn((B * Hq, d), generator=g, device=dev).bfloat16()
        kv = torch.randn((B * Hkv, d), generator=g, device=dev).bfloat16()
        for c in ctxs:
            c.plan()
            c.decode(1, q, kv, kv)
            c.dense_decode(0, q, kv, kv)
    spilled = [c.spill_window().tolist() for c in ctxs]
    assert spilled[0] == spilled[1] and min(spilled[0]) > 0, spilled

    def chunk(c, T_, q, kv, outs=None):
        res = []
        for i, layer in enumerate((1, 0)):
            c.chunk_attend(layer, T_, q, kv, kv, None if outs is None else outs[i])
            res.append(c.last_out_f32())
        return res

    q = torch.randn((B, T, Hq, d), generator=g, device=dev).bfloat16()
    kv = torch.randn((B, T, Hkv, d), generator=g, device=dev).bfloat16()
    got = []
    for c in ctxs:
        c.plan_chunk(T)
        got.append(chunk(c, T, q, kv))
        c.rewind(torch.tensor([(3 * b) % (T + 1) for b in range(B)], dtype=torch.int32, device=dev))
    for layer in range(2):
        err = float((got[0][layer] - got[1][layer]).abs().max())
        assert err <= 1e-5, f"chunk T={T} layer {1 - layer}: shared != twin ({err:.3g})"
    T2 = max(1, T // 3)
    q2, kv2 = q[:, :T2].contiguous(), kv[:, :T2].contiguous()
    sh = ctxs[0]
    sh.plan_chunk(T2)
    eager = chunk(sh, T2, q2, kv2)
    sh.rewind(torch.full((B,), T2, dtype=torch.int32, device=dev))
    outs = [torch.empty((B, T2, Hq * d), dtype=torch.bfloat16, device=dev) for _ in range(2)]
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        sh.plan_chunk(T2)
        chunk(sh, T2, q2, kv2, outs)
    graph.replay()
    torch.cuda.synchronize()
    err = float((sh.last_out_f32() - eager[1]).abs().max())
    assert err <= 1e-5 and sh.error_flags() == 0, f"captured chunk != eager ({err:.3g})"
    print(f"chunk B={B} Hq={Hq} Hkv={Hkv} n={n} T={T} R={R}: ok")


def prefill_case(Hq, Hkv, q_len, kv_len):
    """mpig_prefill_attend at G = Hq / Hkv: the last m-block and the last key tile partial; eager against a torch fp32 restatement
    and a captured launch against the eager one."""
    g = torch.Generator(device=dev).manual_seed(5)
    ctx = Context(6, 24, 1, Hq, Hkv, d, 1, 512, device=dev)
    q = torch.randn((q_len, Hq, d), generator=g, device=dev).bfloat16()
    k = torch.randn((kv_len, Hkv, d), generator=g, device=dev).bfloat16()
    v = torch.randn((kv_len, Hkv, d), generator=g, device=dev).bfloat16()
    f32 = torch.empty((q_len, Hq, d), dtype=torch.float32, device=dev)
    eager = ctx.prefill_attend(q, k, v, out_f32=f32)
    G, off = Hq // Hkv, kv_len - q_len
    s = torch.einsum("thd,khd->htk", q.float(), k.float().repeat_interleave(G, 1)) / d ** 0.5
    vis = torch.arange(kv_len, device=dev)[None] <= off + torch.arange(q_len, device=dev)[:, None]
    ref = torch.einsum("htk,khd->thd", torch.softmax(s.masked_fill(~vis[None], float("-inf")), -1), v.float().repeat_interleave(G, 1))
    err = float((f32 - ref).abs().max() / ref.abs().max())
    assert err <= 1e-3, f"prefill ({q_len}, {kv_len}) G={G}: {err:.3g} from the fp32 restatement"
    out = torch.zeros_like(eager)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ctx.prefill_attend(q, k, v, out)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), eager.view(torch.int16)), "captured prefill != eager"
    print(f"prefill Hq={Hq} Hkv={Hkv} q_len={q_len} kv_len={kv_len}: ok")

if __name__ == "__main__":
    which = sys.argv[1:] or ["stages", "dense", "decode", "hostpeer", "spill", "tokens", "tree", "shared", "shared_spill", "reorder",
                             "chunk", "configs", "compact", "prefill"]
    if "configs" in which:   # BASELINE's C4 and C5 per-rank geometry at small n, each against its decode_impl = 0 twin
        # the i.i.d. keys sampled here have weights near 1e-2, where 1 - (1-p)^(L-1) (Lp + 1 - p) cancels in fp32 and amplifies
        # last-bit differences: the variants differ by up to 4e-4 of a head's largest element at K11 L300 (2e-5 at K10 L150), so
        # they are held to the 1e-3 bar; against fp64 both stay within 2 % of it (tests/test_gpu_config_numerics.py)
        decode_case(1, 32, 8, 3900, 11, 300, tol=1e-3)  # L = 300 over 4 segments: two tag passes, clusters of 4
        decode_case(1, 8, 1, 7900, 10, 150, tol=1e-3)   # one kv-group of 8 heads over 8 segments: clusters of 8
    if "chunk" in which:
        chunk_case(3, 8, 2, 600, 6, 24, 37, 200)      # one key split; T*G = 148: a partial second m-block, partial last tiles
        chunk_case(3, 8, 2, 2100, 6, 24, 5, 200)      # several key splits merged by the last CTA
    if "prefill" in which:
        prefill_case(7, 1, 37, 300)      # 18 tokens per m-block: a partial third m-block; a partial third key tile
        prefill_case(28, 4, 5, 129)      # one m-block of 5 tokens over two key tiles, the second holding one key
    if "compact" in which:
        compact_case(3, 1, 4, 2, 700, 6, 24)
        compact_case(4, 2, 4, 2, 700, 6, 24)             # both slots reclaimed in one call
    if "reorder" in which:
        reorder_case(4, 4, 2, 700, 6, 24, 40)
    if "shared_spill" in which:
        shared_spill_case(3, 4, 2, 700, 6, 24, 3)
    if "shared" in which:
        shared_case(3, 4, 2, 700, 6, 24)                 # clusters of several CTAs per head
    if "tree" in which:
        tree_case(2, 4, 1, 800, 6, 24, [-1, 0, 0, 1, 1, 2], [0, 2, 5])   # clusters of 8 per node, dense T*G = 24 (two m-tiles)
    if "tokens" in which:
        tokens_case(2, 4, 1, 800, 6, 24, 3)              # clusters of 8 per virtual head, dense T*G = 12
        tokens_case(4, 32, 8, 400, 6, 24, 2)             # one CTA per virtual head (codes from the SimHash kernel), dense T*G = 8
    if "spill" in which:
        spill_case()
    if "hostpeer" in which:
        host_and_peer_case()
    if "stages" in which:
        stage_case()
    if "dense" in which:
        dense_case()
    if "decode" in which:
        decode_case(1, 4, 2, 600, 6, 24)                 # cluster of 8 CTAs per head
        decode_case(1, 8, 2, 3000, 6, 40, selcap=16)     # several selection passes
        decode_case(1, 4, 1, 66000, 8, 20)               # two key segments (cluster 2 x 4)
        decode_case(4, 32, 8, 500, 6, 24)                # 128 heads: one CTA per head, codes from the SimHash kernel
        decode_case(5, 32, 8, 400, 6, 24)                # 160 heads: two 512-thread CTAs per SM
        decode_case(1, 4, 2, 900, 9, 300)                # more tables than one-byte tag ids: two tag passes in the fused kernel
    print("ALL OK")
