"""Window spill (mpig_spill_window, `-m gpu`): generated tokens leave the sink + local + generated window for the sampled store
and the hash tables, so a generation can run past generation_buffer.

  * the tables after a spill equal a device rebuild over all keys (offsets identical, items equal as a set per bucket);
  * spilled records are the window rows bit for bit, their norms within one bf16 ulp of torch's;
  * a decode after a spill matches the oracle fed the server's own stored state, and samples spilled keys;
  * a decode step captured before a spill stays valid after it;
  * the drop-in class generates 3 x generation_buffer + 5 tokens;
  * a refused spill changes nothing.
"""
import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200 import synth
from tests.support.fp64 import assert_1e3_f32, oracle_decode
from tests.support.library import DEV, NL, NS, Run, _Cfg, assert_tables_equal, d, lsh_tables

pytestmark = pytest.mark.gpu


def _segment_len(ctx):
    o, _ = lsh_tables(ctx, 1)
    assert o.shape[3] >= 2, "shape must have two key segments"
    return int(o[0, 0, 0, 1, 0])


@pytest.mark.parametrize("route", ["build", "sorted"])
@pytest.mark.parametrize("B,Hq,Hkv,n,K,L,M,gen,steps,straddle", [
    (2, 8, 2, 1500, 8, 40, 2048, 40, 30, False),
    (1, 4, 1, 1000, 7, 24, 4096, 64, 50, True),        # 4 segments of 1024 keys: the spill straddles 1024
    (1, 4, 2, 2000, 15, 8, 4096, 32, 20, False),       # K = 15: the merge reads the old offsets from HBM
])
def test_tables_equal_rebuild(cuda_lib, route, B, Hq, Hkv, n, K, L, M, gen, steps, straddle):
    r = Run(B, Hq, Hkv, n, K, L, M, gen, seed=n + K, route=route)
    for _ in range(steps):
        _, k, v, _ = r.token()
        r.push(k, v)
    n_old = r.n_off
    g, (sk, sv) = r.spill()
    assert g == steps
    if straddle:
        seg_len = _segment_len(r.ctx)
        assert any(n_old < s * seg_len < n_old + g for s in range(1, M // seg_len + 1)), "spill should straddle a segment"
    assert_tables_equal(lsh_tables(r.ctx, 1), lsh_tables(r.rebuild(), 1), range(B))
    # store: spilled records are the window rows bit for bit, norms within one bf16 ulp of torch's norm of them
    k_st, v_st, kn_st = (x.cpu() for x in r.ctx.read_cache(1))
    assert torch.equal(k_st[:, :, n_old:n_old + g].view(torch.int16), sk.contiguous().view(torch.int16))
    assert torch.equal(v_st[:, :, n_old:n_old + g].view(torch.int16), sv.contiguous().view(torch.int16))
    ref = k_st[:, :, n_old:n_old + g].to(DEV).norm(p=2, dim=-1).float().cpu()
    got = kn_st[:, :, n_old:n_old + g]
    assert torch.equal(got.bfloat16().float(), got), "norms are bf16 values"
    assert float(((got - ref).abs() / ref.abs().clamp_min(1e-30)).max()) <= 2 ** -7
    # the original keys are untouched
    assert torch.equal(k_st[:, :, :n].view(torch.int16), r.key.view(torch.int16))
    # two spills in a row: 12 more tokens, then a spill moves exactly 12 (the window length was sink + keep)
    for _ in range(12):
        _, k, v, _ = r.token()
        r.push(k, v)
    g2, _ = r.spill()
    assert g2 == 12
    assert_tables_equal(lsh_tables(r.ctx, 1), lsh_tables(r.rebuild(), 1), range(B))


def test_tables_equal_rebuild_c2(cuda_lib):
    """C2 (Llama-3.1-8B, P = 98 000, M = 98 304): a full window of 324 rows spills g = 256 keys."""
    P, M = 98000, 98304
    n = P - NS - NL
    r = Run(1, 32, 8, n, 10, 150, M, 256, seed=7, on_gpu=True, w0=NS + NL + 250)
    for _ in range(6):
        _, k, v, _ = r.token()
        r.push(k, v)
    assert r.wk.shape[2] == 324
    g, _ = r.spill()
    assert g == 256
    assert_tables_equal(lsh_tables(r.ctx, 1), lsh_tables(r.rebuild(), 1), [0])


def test_decode_after_spill(cuda_lib):
    """Both decode variants (fused and three launches) after a spill, against the oracle and against each other."""
    B, Hq, Hkv, n, K, L = 2, 8, 2, 1500, 6, 40
    got = {}
    for which in (1, 0):
        r = Run(B, Hq, Hkv, n, K, L, 2048, 48, seed=11, impl=which)
        r.ctx.set_option("save_mask", 1)
        for _ in range(40):
            _, k, v, _ = r.token()
            r.push(k, v)
        n_old = r.n_off
        g, (sk, _) = r.spill()
        # queries near spilled keys (cos ~ 0.97): those keys collide in most tables and must be sampled
        noise = torch.randn((B, Hq, 1, d), generator=torch.Generator().manual_seed(12)) * 0.25
        q = (sk[:, :, 5:6].float().repeat_interleave(r.G, dim=1) + noise).bfloat16()
        q, k, v, out = r.token(q)
        o32 = r.ctx.last_out_f32().cpu()
        nnz, res = r.ctx.last_probe(want_results=True)
        r.check_decode(q, k, v, o32)
        nnz, res = nnz.cpu(), res.cpu()
        sel = [res[h, : nnz[h]] for h in range(B * Hq)]
        assert all(int((s >= n_old).sum()) > 0 for s in sel), "spilled keys are never sampled"
        assert all(int(s.max()) < n_old + g for s in sel if len(s))
        got[which] = sel
        r.push(k, v)
    for a, b in zip(got[0], got[1]):
        assert torch.equal(a, b), "fused and three-launch decodes select different keys"


def test_captured_step_survives_spill(cuda_lib):
    B, Hq, Hkv, n, K, L = 1, 8, 2, 1200, 7, 30
    outs = {}
    for mode in ("eager", "graph"):
        r = Run(B, Hq, Hkv, n, K, L, 2048, 16, seed=13)
        qs, ks, vs = (torch.zeros(s, dtype=torch.bfloat16, device=DEV) for s in ((B, Hq, 1, d), (B, Hkv, 1, d), (B, Hkv, 1, d)))
        out = torch.zeros((B, Hq * d), dtype=torch.bfloat16, device=DEV)
        g = torch.Generator().manual_seed(99)
        seq = [tuple(torch.randn(s, generator=g).bfloat16() for s in ((B, Hq, 1, d), (B, Hkv, 1, d), (B, Hkv, 1, d)))
               for _ in range(40)]
        r.ctx.plan()   # the same eager first token in both modes (also the warm-up before a capture)
        r.ctx.decode(1, qs, ks, vs, out)
        step = None
        if mode == "graph":
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            gph = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s):
                with torch.cuda.graph(gph, stream=s):
                    r.ctx.plan()
                    r.ctx.decode(1, qs, ks, vs, out)
            torch.cuda.current_stream().wait_stream(s)
            step = gph.replay
        else:
            def step():
                r.ctx.plan()
                r.ctx.decode(1, qs, ks, vs, out)
        res = []
        used = 1
        for q, k, v in seq:
            if used == 16:
                torch.cuda.synchronize()
                assert r.ctx.spill_window().tolist() == [16]
                used = 0
            qs.copy_(q.to(DEV)), ks.copy_(k.to(DEV)), vs.copy_(v.to(DEV))
            step()
            used += 1
            res.append(out.clone())
        torch.cuda.synchronize()
        assert r.ctx.error_flags() == 0
        outs[mode] = torch.stack(res).cpu()
    assert torch.equal(outs["eager"].view(torch.int16), outs["graph"].view(torch.int16))


def test_long_generation_dropin(cuda_lib):
    from magicpig_b200.attnserver import LSHSparseAttnServer
    cfg = _Cfg()
    K, L, B, P, M, gen = 6, 40, 2, 600, 1024, 16
    Hq, Hkv, G = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.num_attention_heads // cfg.num_key_value_heads
    g = torch.Generator().manual_seed(17)
    hf = synth.make_hash_func(d, K, L, seed=18)
    srv = LSHSparseAttnServer(cfg, K=K, L=L, batch_size=B, max_length=M, generation_buffer=gen, dense_layers=[0, 16],
                              device=DEV, hash_func=hf)
    srv.ctx.set_option("out_f32", 1)
    kcs = [torch.randn((B, M, Hkv, d), generator=g).bfloat16() for _ in range(3)]
    vcs = [torch.randn((B, M, Hkv, d), generator=g).bfloat16() for _ in range(3)]
    srv.alloc_buffer(P)
    for b in range(B):
        for layer in range(3):
            srv.fill(layer, b, kcs[layer][b].to(DEV), vcs[layer][b].to(DEV), P)
            srv.build_table(layer, b, P)
    layer = 2
    avg = srv.avg_k[layer].cpu()
    kc, vc = kcs[layer][:, :P].transpose(1, 2), vcs[layer][:, :P].transpose(1, 2)
    wk = torch.cat([kc[:, :, :NS], kc[:, :, P - NL:P]], dim=2) - avg
    wv = torch.cat([vc[:, :, :NS], vc[:, :, P - NL:P]], dim=2)
    n_off, used = P - NS - NL, 0
    steps = 3 * gen + 5
    for i in range(steps):
        if used == gen:   # the next plan() would find the window full
            spilled = srv.spill_window()
            assert spilled.tolist() == [gen] * B
            wk = torch.cat([wk[:, :, :NS], wk[:, :, NS + gen:]], dim=2)
            wv = torch.cat([wv[:, :, :NS], wv[:, :, NS + gen:]], dim=2)
            n_off += gen
            used = 0
        q = torch.randn((B, Hq, 1, d), generator=g).bfloat16()
        k_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
        v_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
        srv.plan()
        used += 1
        for lyr in range(3):   # layer 2 last: last_probe / last_out_f32 are its
            srv.decode(q.to(DEV), k_new.to(DEV), v_new.to(DEV), lyr)
        if i < steps - 1:
            wk = torch.cat([wk, k_new - avg], dim=2)
            wv = torch.cat([wv, v_new], dim=2)
    assert srv.ctx.error_flags() == 0
    assert n_off == P - NS - NL + 3 * gen
    # the last step against the oracle fed the stored state of layer 2
    o32 = srv.ctx.last_out_f32().cpu()
    nnz = srv.ctx.last_probe()[0].cpu()
    k_st, v_st, kn_st = (x.cpu() for x in srv.ctx.read_cache(layer))
    kk = k_st[:, :, :n_off].contiguous()
    kcodes = torch.stack([srv.ctx.hash_keys(kk[b].to(DEV)).cpu() for b in range(B)])
    t = dict(B=B, Hq=Hq, Hkv=Hkv, d=d, K=K, L=L, n=n_off, M=M, hash_func=hf, kcodes=kcodes, key=kk,
             value=v_st[:, :, :n_off].contiguous(), key_norm=kn_st[:, :, :n_off].contiguous(), avg_k=avg)
    _, nz_ref, _, o_exact = oracle_decode(t, q, k_new, v_new, wk, wv, G)
    assert torch.equal(nnz, nz_ref)
    assert_1e3_f32(o32, o_exact)
    srv.clear()

def _snapshot(ctx):
    o, i = lsh_tables(ctx, 1)
    k, v, kn = ctx.read_cache(1)
    return [o, i, k.view(torch.int16), v.view(torch.int16), kn]


def _unchanged(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def test_refused_spill_changes_nothing(cuda_lib):
    # max_length: 20 generated rows do not fit beside 1000 keys in M = 1010
    r = Run(1, 4, 2, 1000, 6, 16, 1010, 24, seed=21)
    for _ in range(20):
        _, k, v, _ = r.token()
        r.push(k, v)
    before = _snapshot(r.ctx)
    with pytest.raises(N.MagicPigError, match=r"code -4.*max_length"):
        r.ctx.spill_window()
    for bad in (-1, 24 + NL):   # sink + keep >= window capacity (4 + 64 + 24)
        with pytest.raises(N.MagicPigError, match="code -1"):
            r.ctx.spill_window(bad)
    assert _unchanged(before, _snapshot(r.ctx))
    # the window length is unchanged too: keeping 78 rows spills exactly the 10 that fit
    assert r.ctx.spill_window(NL + 10).tolist() == [10]
    # no hash_func: the spilled keys cannot be hashed
    from magicpig_b200.ops import Context
    ctx = Context(6, 16, 2, 4, 2, d, 1, 2048, NS, NL, 24, dense_layers=[0], device=DEV)
    key, value, kn, avg = synth.make_kv(1, 2, 500, d, seed=22)
    hf = synth.make_hash_func(d, 6, 16, seed=23)
    ctx.attn_fill(1, 0, key[0].to(DEV), value[0].to(DEV), kn[0].to(DEV))
    ctx.lsh_build(1, 0, synth.hash_keys(key[0], hf, 6, 16).to(DEV))
    wk = torch.randn((2, NS + NL + 12, d)).bfloat16()
    ctx.window_fill(1, 0, avg[0].reshape(2, d).to(DEV), wk.to(DEV), wk.to(DEV))
    before = _snapshot(ctx)
    with pytest.raises(N.MagicPigError, match=r"code -4.*hash_func"):
        ctx.spill_window()
    assert _unchanged(before, _snapshot(ctx))
    ctx.set_hash_func(hf.to(DEV))
    assert ctx.spill_window().tolist() == [12]
