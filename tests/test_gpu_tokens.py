"""Verification steps of T tokens (`-m gpu`): mpig_plan_tokens -> mpig_decode_tokens / mpig_dense_decode_tokens -> mpig_rewind.

A step of T tokens must equal T single-token steps on the same inputs:
  * sparse layers: identical query codes, nnz and index lists, fp32 outputs within 1e-5, each token within 1e-3 of the oracle
    fed the window rows up to its position, and the bf16 output = the fp32 output rounded once;
  * dense layers: within 1e-5 of T sequential dense decodes and 1e-3 of an fp64 causal restatement;
  * a rewind leaves the state of a twin that decoded only the accepted tokens; a captured plan -> layers -> rewind replays with
    changing drops; multi-token steps run into a spill; every refusal leaves the state unchanged.
"""
import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200 import synth
from tests.support.fp64 import assert_1e3_f32, assert_rounded_half_up, oracle_decode, rel_max
from tests.support.library import DEV, NL, NS, Run, Twins, _Cfg, assert_tables_equal, d, lsh_tables

pytestmark = pytest.mark.gpu


def run_sparse_step(tw, T, q, k, v):
    """One T-token step on `tok` and T single steps on `seq`; returns both sides' (out, o32, nnz, res, codes), (B, T, Hq, ...)."""
    B, Hq = tw.B, tw.Hq
    tw.tok.plan(T)
    out = tw.tok.decode_tokens(1, T, q.to(DEV), k.to(DEV), v.to(DEV)).cpu().reshape(B, T, Hq, d)
    nnz, res = tw.tok.last_probe(want_results=True)
    a = dict(out=out, o32=tw.tok.last_out_f32().cpu().reshape(B, T, Hq, d), nnz=nnz.cpu().reshape(B, T, Hq),
             res=res.cpu().reshape(B, T, Hq, -1), codes=tw.tok.last_codes().cpu().reshape(B, T, Hq, -1))
    s = {key: [] for key in a}
    for t in range(T):
        tw.seq.plan()
        o = tw.seq.decode(1, q[:, t].contiguous().to(DEV), k[:, t].contiguous().to(DEV), v[:, t].contiguous().to(DEV))
        nz, rs = tw.seq.last_probe(want_results=True)
        s["out"].append(o.cpu().reshape(B, Hq, d))
        s["o32"].append(tw.seq.last_out_f32().cpu().reshape(B, Hq, d))
        s["nnz"].append(nz.cpu().reshape(B, Hq))
        s["res"].append(rs.cpu().reshape(B, Hq, -1))
        s["codes"].append(tw.seq.last_codes().cpu().reshape(B, Hq, -1))
    s = {key: torch.stack(x, dim=1) for key, x in s.items()}
    return a, s


def assert_same_as_sequential(a, s):
    assert torch.equal(a["codes"], s["codes"])
    assert torch.equal(a["nnz"], s["nnz"])
    B, T, Hq = a["nnz"].shape
    for b in range(B):
        for t in range(T):
            for h in range(Hq):
                n_ = int(a["nnz"][b, t, h])
                assert torch.equal(a["res"][b, t, h, :n_], s["res"][b, t, h, :n_]), (b, t, h)
    assert rel_max(a["o32"], s["o32"]) <= 1e-5
    assert_rounded_half_up(a["out"], a["o32"], "T-token step")


@pytest.mark.parametrize("T", [2, 3, 8])
@pytest.mark.parametrize("B,Hq,Hkv,n,K,L", [
    (2, 16, 4, 4096, 10, 150),     # clusters of 4
    (2, 4, 1, 1500, 8, 60),        # clusters of 8
    (2, 4, 1, 70000, 8, 40),       # two key segments
    (4, 32, 8, 2000, 8, 60),       # 128 heads, one CTA each (codes from the stand-alone SimHash kernel)
    (5, 32, 8, 1200, 8, 40),       # 160 heads: 512-thread CTAs
])
def test_sparse_tokens_match_sequential(cuda_lib, B, Hq, Hkv, n, K, L, T):
    tw = Twins(B, Hq, Hkv, n, K, L, T, seed=n + T)
    q, k, v = tw.inputs(T)
    a, s = run_sparse_step(tw, T, q, k, v)
    assert_same_as_sequential(a, s)
    assert tw.tok.get_info("tokens_cluster_waves") >= 1
    if T == 8 and B * Hq >= 128:
        assert tw.tok.get_info("tokens_cluster_waves") >= 2, "shape should need several waves"
    if n > 5000 or K >= 10:
        # (at K10 L150 the single-token decode itself sits at the 1e-3 bar on these random queries; the tokens equal it above)
        return
    # every token against the oracle, fed the window rows up to its position
    for b in range(B):
        tb = dict(B=1, Hq=Hq, Hkv=Hkv, d=d, K=K, L=L, n=n, M=tw.M, hash_func=tw.hf, kcodes=tw.kcodes[b:b + 1],
                  key=tw.key[b:b + 1], value=tw.value[b:b + 1], key_norm=tw.kn[b:b + 1], avg_k=tw.avg[b:b + 1])
        wk, wv = tw.win[b][0][None], tw.win[b][1][None]
        for t in range(T):
            kt, vt = k[b:b + 1, t][:, :, None], v[b:b + 1, t][:, :, None]
            _, nz_ref, _, o_exact = oracle_decode(tb, q[b:b + 1, t][:, :, None], kt, vt, wk, wv, tw.G)
            assert torch.equal(a["nnz"][b, t], nz_ref)
            assert_1e3_f32(a["o32"][b, t], o_exact)
            wk = torch.cat([wk, kt - tw.avg[b:b + 1]], dim=2)
            wv = torch.cat([wv, vt], dim=2)


def test_sparse_tokens_c2_size(cuda_lib):
    """Llama-3.1-8B shape at P = 98 000 (K10 L150, B = 1): a step of 4 tokens against 4 single steps."""
    P = 98000
    tw = Twins(1, 32, 8, P - NS - NL, 10, 150, 4, seed=3, on_gpu=True)
    q, k, v = tw.inputs(4)
    a, s = run_sparse_step(tw, 4, q, k, v)
    assert_same_as_sequential(a, s)


@pytest.mark.parametrize("B,Hq,Hkv,P,T", [(2, 8, 2, 777, 3), (2, 8, 2, 777, 2), (2, 8, 2, 777, 4), (1, 8, 1, 5000, 4),
                                          (3, 4, 4, 31, 8), (1, 32, 8, 20000, 8)])
def test_dense_tokens(cuda_lib, B, Hq, Hkv, P, T):
    """T*G query rows per kv-group: 8 (hi/lo packed in one m-tile), 12 / 16 (one m-tile), 32 (two m-tiles)."""
    tw = Twins(B, Hq, Hkv, 64, 4, 8, T, seed=P + T, P_dense=P)
    G = Hq // Hkv
    q, k, v = tw.inputs(T)
    tw.tok.plan(T)
    out = tw.tok.dense_decode_tokens(0, T, q.to(DEV), k.to(DEV), v.to(DEV)).cpu().reshape(B, T, Hq, d)
    o32 = tw.tok.last_out_f32().cpu().reshape(B, T, Hq, d)
    seq = []
    for t in range(T):
        tw.seq.plan()
        tw.seq.dense_decode(0, q[:, t].contiguous().to(DEV), k[:, t].contiguous().to(DEV), v[:, t].contiguous().to(DEV))
        seq.append(tw.seq.last_out_f32().cpu().reshape(B, Hq, d))
    assert rel_max(o32, torch.stack(seq, dim=1)) <= 1e-5
    assert_rounded_half_up(out, o32, "dense T-token step")
    # fp64 causal restatement
    kk = torch.cat([tw.dk, k], dim=1).double()   # (B, P+T, Hkv, d)
    vv = torch.cat([tw.dv, v], dim=1).double()
    for t in range(T):
        n_vis = P + t + 1
        qt = q[:, t].double().reshape(B, Hkv, G, d)
        s_ = torch.einsum("bkgd,bnkd->bkgn", qt, kk[:, :n_vis]) / d ** 0.5
        ref = torch.einsum("bkgn,bnkd->bkgd", torch.softmax(s_, dim=-1), vv[:, :n_vis]).reshape(B * Hq, d)
        assert_1e3_f32(o32[:, t].reshape(B * Hq, d), ref)


def single_request_twin(tw, b):
    """A B = 1 context holding exactly request b of `tw` (same keys, tables, window and dense rows)."""
    from magicpig_b200.ops import Context
    ctx = Context(tw.K, tw.L, 2, tw.Hq, tw.Hkv, d, 1, tw.M, NS, NL, 32, dense_layers=[0], alloc_dense_kv=True, device=DEV,
                  max_query_tokens=2)
    ctx.set_option("out_f32", 1)
    ctx.set_hash_func(tw.hf.to(DEV))
    ctx.attn_fill(1, 0, tw.key[b].to(DEV).contiguous(), tw.value[b].to(DEV).contiguous(), tw.kn[b].to(DEV).contiguous())
    ctx.lsh_build(1, 0, tw.kcodes[b].to(DEV))
    ctx.window_fill(1, 0, tw.avg[b].reshape(tw.Hkv, d).to(DEV), tw.win[b][0].to(DEV), tw.win[b][1].to(DEV))
    ctx.dense_fill(0, 0, tw.dk[b].to(DEV), tw.dv[b].to(DEV), tw.dk.shape[1])
    return ctx


def test_rewind_equals_accepted_only(cuda_lib):
    """T = 4 with drop = [3, 1]: both layers then behave like twins that decoded only the accepted tokens (1 and 3, one at a
    time): the same nnz and outputs on the next steps (one of 1 token, one of 2)."""
    B, Hq, Hkv, n, K, L, T = 2, 8, 2, 1500, 8, 40, 4
    tw = Twins(B, Hq, Hkv, n, K, L, T, seed=77)
    q, k, v = tw.inputs(T)
    tw.tok.plan(T)
    tw.tok.decode_tokens(1, T, q.to(DEV), k.to(DEV), v.to(DEV))
    tw.tok.dense_decode_tokens(0, T, q.to(DEV), k.to(DEV), v.to(DEV))
    tw.tok.rewind(torch.tensor([3, 1], dtype=torch.int32, device=DEV))
    twins = []
    for b, acc in ((0, 1), (1, 3)):
        c = single_request_twin(tw, b)
        for t in range(acc):
            c.plan()
            c.decode(1, q[b:b + 1, t].contiguous().to(DEV), k[b:b + 1, t].contiguous().to(DEV), v[b:b + 1, t].contiguous().to(DEV))
            c.dense_decode(0, q[b:b + 1, t].contiguous().to(DEV), k[b:b + 1, t].contiguous().to(DEV), v[b:b + 1, t].contiguous().to(DEV))
        twins.append(c)
    for T2 in (1, 2):
        q2, k2, v2 = tw.inputs(T2)
        tw.tok.plan(T2)
        tw.tok.decode_tokens(1, T2, q2.to(DEV), k2.to(DEV), v2.to(DEV))
        o_s = tw.tok.last_out_f32().cpu().reshape(B, T2, Hq, d)
        nz = tw.tok.last_probe()[0].cpu().reshape(B, T2, Hq)
        tw.tok.dense_decode_tokens(0, T2, q2.to(DEV), k2.to(DEV), v2.to(DEV))
        o_d = tw.tok.last_out_f32().cpu().reshape(B, T2, Hq, d)
        for b, c in enumerate(twins):
            args = (q2[b:b + 1].contiguous().to(DEV), k2[b:b + 1].contiguous().to(DEV), v2[b:b + 1].contiguous().to(DEV))
            c.plan(T2)
            c.decode_tokens(1, T2, *args)
            assert torch.equal(c.last_probe()[0].cpu().reshape(T2, Hq), nz[b])
            assert rel_max(o_s[b], c.last_out_f32().cpu().reshape(T2, Hq, d)) <= 1e-5
            c.dense_decode_tokens(0, T2, *args)
            assert rel_max(o_d[b], c.last_out_f32().cpu().reshape(T2, Hq, d)) <= 1e-5


def test_graph_replay_with_changing_drops(cuda_lib):
    """plan(T) -> sparse + dense layers -> rewind(device drops), captured once and replayed with new inputs and drops, equals an
    eager twin; a single-token step captured before stays valid."""
    B, Hq, Hkv, n, K, L, T = 2, 8, 2, 1500, 8, 40, 3
    tw = Twins(B, Hq, Hkv, n, K, L, T, seed=31, gen=64)
    eager = Twins(B, Hq, Hkv, n, K, L, T, seed=31, gen=64).tok
    ctx = tw.tok
    q_s = torch.zeros((B, T, Hq, d), dtype=torch.bfloat16, device=DEV)
    k_s = torch.zeros((B, T, Hkv, d), dtype=torch.bfloat16, device=DEV)
    v_s = torch.zeros_like(k_s)
    q1 = torch.zeros((B, 1, Hq, d), dtype=torch.bfloat16, device=DEV)
    k1 = torch.zeros((B, 1, Hkv, d), dtype=torch.bfloat16, device=DEV)
    v1 = torch.zeros_like(k1)
    drop_s = torch.zeros(B, dtype=torch.int32, device=DEV)
    out_s = torch.empty((B, T, Hq * d), dtype=torch.bfloat16, device=DEV)
    out_d = torch.empty_like(out_s)
    out1 = torch.empty((B, 1, Hq * d), dtype=torch.bfloat16, device=DEV)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    g1, gT = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        ctx.plan(1)   # warm-up outside capture (plans are cached per T)
        ctx.decode_tokens(1, 1, q1, k1, v1, out1)
        ctx.rewind(torch.ones(B, dtype=torch.int32, device=DEV))
        ctx.plan(T)
        ctx.decode_tokens(1, T, q_s, k_s, v_s, out_s)
        ctx.rewind(torch.full((B,), T, dtype=torch.int32, device=DEV))
        with torch.cuda.graph(g1, stream=st):
            ctx.plan(1)
            ctx.decode_tokens(1, 1, q1, k1, v1, out1)
        with torch.cuda.graph(gT, stream=st):
            ctx.plan(T)
            ctx.decode_tokens(1, T, q_s, k_s, v_s, out_s)
            ctx.dense_decode_tokens(0, T, q_s, k_s, v_s, out_d)
            ctx.rewind(drop_s)
    torch.cuda.current_stream().wait_stream(st)
    torch.cuda.synchronize()
    for it, drops in enumerate(([1, 0], [0, 2], [3, 1], [2, 2])):
        q, k, v = tw.inputs(T)
        q_s.copy_(q), k_s.copy_(k), v_s.copy_(v)
        drop_s.copy_(torch.tensor(drops, dtype=torch.int32))
        gT.replay()
        torch.cuda.synchronize()
        eager.plan(T)
        e_s = eager.decode_tokens(1, T, q.to(DEV), k.to(DEV), v.to(DEV)).cpu()
        e_d = eager.dense_decode_tokens(0, T, q.to(DEV), k.to(DEV), v.to(DEV)).cpu()
        eager.rewind(torch.tensor(drops, dtype=torch.int32, device=DEV))
        assert torch.equal(out_s.cpu(), e_s), it
        assert torch.equal(out_d.cpu(), e_d), it
        # the single-token graph captured earlier
        qq, kk, vv = tw.inputs(1)
        q1.copy_(qq), k1.copy_(kk), v1.copy_(vv)
        g1.replay()
        torch.cuda.synchronize()
        eager.plan(1)
        e1 = eager.decode_tokens(1, 1, qq.to(DEV), kk.to(DEV), vv.to(DEV)).cpu()
        assert torch.equal(out1.cpu(), e1), it
    assert ctx.error_flags() == 0


def test_tokens_then_spill(cuda_lib):
    """Steps of 4 tokens with rewinds until the window is full, then a spill: the tables equal a rebuild, and a 4-token step after
    the spill matches the oracle token by token."""
    B, Hq, Hkv, n, K, L, gen = 2, 8, 2, 1500, 8, 40, 24
    r = Run(B, Hq, Hkv, n, K, L, 2048, gen, seed=5)
    r.ctx.reserve_query_tokens(4)
    r.ctx.set_option("save_mask", 1)

    def step(drop):
        q = torch.randn((B, 4, Hq, d), generator=r.g).bfloat16()
        k = torch.randn((B, 4, Hkv, d), generator=r.g).bfloat16()
        v = torch.randn((B, 4, Hkv, d), generator=r.g).bfloat16()
        r.ctx.plan(4)
        r.ctx.decode_tokens(1, 4, q.to(DEV), k.to(DEV), v.to(DEV))
        o32 = r.ctx.last_out_f32().cpu().reshape(B, 4, Hq, d)
        nnz = r.ctx.last_probe()[0].cpu().reshape(B, 4, Hq)
        r.ctx.rewind(torch.full((B,), drop, dtype=torch.int32, device=DEV))
        return q, k, v, o32, nnz

    used = 0
    for drop in (1, 3, 0, 2, 1, 0, 2, 3, 1, 0, 2):
        if used + 4 > gen:
            break
        q, k, v, _, _ = step(drop)
        for t in range(4 - drop):
            r.push(k[:, t][:, :, None], v[:, t][:, :, None])
        used += 4 - drop
    g, _ = r.spill()
    assert g == used
    assert_tables_equal(lsh_tables(r.ctx, 1), lsh_tables(r.rebuild(), 1), range(B))
    q, k, v, o32, nnz = step(0)
    for t in range(4):
        qt, kt, vt = q[:, t][:, :, None], k[:, t][:, :, None], v[:, t][:, :, None]
        n_ = r.n_off
        k_st, v_st, kn_st = (x.cpu() for x in r.ctx.read_cache(1))
        kcodes = torch.stack([r.ctx.hash_keys(k_st[b, :, :n_].contiguous().to(DEV)).cpu() for b in range(B)])
        tdict = dict(B=B, Hq=Hq, Hkv=Hkv, d=d, K=K, L=L, n=n_, M=r.M, hash_func=r.hf, kcodes=kcodes, key=k_st[:, :, :n_].contiguous(),
                     value=v_st[:, :, :n_].contiguous(), key_norm=kn_st[:, :, :n_].contiguous(), avg_k=r.avg)
        _, nz_ref, _, o_exact = oracle_decode(tdict, qt, kt, vt, r.wk, r.wv, r.G)
        assert torch.equal(nnz[:, t].reshape(-1), nz_ref)
        assert_1e3_f32(o32[:, t].reshape(B * Hq, d), o_exact)
        r.push(kt, vt)


def test_tokens_refusals(cuda_lib):
    from magicpig_b200.ops import Context
    B, Hq, Hkv, T = 2, 8, 2, 4
    tw = Twins(B, Hq, Hkv, 1500, 8, 40, T, seed=9, gen=8)
    ctx = tw.tok
    q, k, v = tw.inputs(T)
    qd, kd, vd = q.to(DEV), k.to(DEV), v.to(DEV)
    # T = 1 through decode_tokens is bitwise decode()
    q1, k1, v1 = tw.inputs(1)
    ctx.plan()
    a = ctx.decode_tokens(1, 1, q1.to(DEV), k1.to(DEV), v1.to(DEV)).cpu()
    tw.seq.plan()
    b_ = tw.seq.decode(1, q1.to(DEV), k1.to(DEV), v1.to(DEV)).cpu()
    assert torch.equal(a.reshape(-1), b_.reshape(-1))
    with pytest.raises(N.MagicPigError, match="outside"):
        ctx.plan(T + 1)                                                     # more than reserved
    with pytest.raises(N.MagicPigError, match="last plan"):
        ctx.decode_tokens(1, T, qd, kd, vd)                                 # planned for 1 token
    ctx.plan(T)
    with pytest.raises(N.MagicPigError, match="last plan"):
        ctx.decode_tokens(1, 2, qd[:, :2].contiguous(), kd[:, :2].contiguous(), vd[:, :2].contiguous())
    ctx.set_option("decode_impl", 0)
    with pytest.raises(N.MagicPigError, match="decode_impl"):
        ctx.decode_tokens(1, T, qd, kd, vd)
    ctx.set_option("decode_impl", 1)
    with pytest.raises(N.MagicPigError, match="outside"):
        ctx.rewind(torch.tensor([T + 1, -1], dtype=torch.int32, device=DEV))   # bad drops: nothing changes, bit 2
    assert ctx.error_flags() & 4
    ctx.rewind(torch.zeros(B, dtype=torch.int32, device=DEV))               # the refused rewind may be repeated
    with pytest.raises(N.MagicPigError, match="at most one rewind"):
        ctx.rewind(torch.zeros(B, dtype=torch.int32, device=DEV))
    # the lengths are those of the plan (the bad rewind changed nothing): the window takes gen - 1 - T more tokens, then refuses
    left = 8 - 1 - T
    ctx.plan(left) if left > 1 else ctx.plan()
    with pytest.raises(N.MagicPigError, match="window is full"):
        ctx.plan()                                                          # plan overflow refused before anything changes
    ctx.rewind(torch.full((B,), left, dtype=torch.int32, device=DEV))
    ctx.plan()
    # T*G > 32 on a dense layer
    big = Context(4, 8, 1, 32, 4, d, 1, 512, dense_layers=[0], alloc_dense_kv=True, device=DEV, max_query_tokens=8)
    big.dense_fill(0, 0, torch.zeros((10, 4, d), dtype=torch.bfloat16, device=DEV),
                   torch.zeros((10, 4, d), dtype=torch.bfloat16, device=DEV), 10)
    big.plan(8)
    z = torch.zeros((1, 8, 32, d), dtype=torch.bfloat16, device=DEV)
    zk = torch.zeros((1, 8, 4, d), dtype=torch.bfloat16, device=DEV)
    with pytest.raises(N.MagicPigError, match="at most 32"):
        big.dense_decode_tokens(0, 8, z, zk, zk)
    assert big.get_info("query_tokens_max") == 8
    assert ctx.get_info("query_tokens_max") == T
    # clear() forgets the pending step and the row count of the readers
    ctx.clear()
    ctx.plan(T)
    ctx.decode_tokens(1, T, qd, kd, vd)
    assert ctx.last_probe()[0].numel() == B * T * Hq
    ctx.clear()
    assert ctx.last_probe()[0].numel() == B * Hq and int(ctx.last_probe()[0].abs().sum()) == 0
    with pytest.raises(N.MagicPigError, match="at most one rewind"):
        ctx.rewind(torch.zeros(B, dtype=torch.int32, device=DEV))
    # the scratch cannot move once a step has been captured
    s_ = torch.cuda.Stream()
    s_.wait_stream(torch.cuda.current_stream())
    gph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s_):
        with torch.cuda.graph(gph, stream=s_):
            tw.seq.plan()
    torch.cuda.synchronize()
    with pytest.raises(N.MagicPigError, match="reserve before capturing"):
        tw.seq.reserve_query_tokens(4)


def test_runner_step_tokens_matches_single_steps(cuda_lib):
    """LlamaDecodeRunner.step_tokens(T) on a 2-layer model (one dense, one sparse layer): the logits after each of the T tokens
    match T single-token eager steps of a twin runner, and so does the next step."""
    from magicpig_b200.llama_runner import LlamaDecodeRunner, LlamaShape
    shape = LlamaShape("tiny", 2, 512, 1024, 4, 2, 1000, 500000.0, 1e-5)
    B, P, T = 2, 300, 3
    runners = [LlamaDecodeRunner(shape, 6, 16, B, 1024, seed=3, generation_buffer=32, dense_layers=(0,), fused=False,
                                 max_query_tokens=T) for _ in range(2)]
    for r in runners:
        r.synthetic_prefill(P, seed=9)
    spec, twin = runners
    ids = torch.randint(0, shape.vocab_size, (B, T), generator=torch.Generator().manual_seed(4)).to(DEV)
    spec.ids_tok[:, :T].copy_(ids)
    got = spec.step_tokens(T, drop=torch.zeros(B, dtype=torch.int32, device=DEV)).clone()
    ref = []
    for t in range(T):
        twin.ids.copy_(ids[:, t:t + 1])
        ref.append(twin.step().clone())
    ref = torch.stack(ref, dim=1)
    assert rel_max(got, ref) <= 2e-2      # bf16 GEMMs over B*T rows against B rows
    assert torch.equal(spec.pos.cpu(), twin.pos.cpu())
    nxt = torch.randint(0, shape.vocab_size, (B, 1), generator=torch.Generator().manual_seed(5)).to(DEV)
    spec.ids_tok[:, :1].copy_(nxt)
    a = spec.step_tokens(1).clone()
    twin.ids.copy_(nxt)
    b_ = twin.step().clone()
    assert rel_max(a[:, 0], b_) <= 2e-2


def test_dropin_speculative_loop(cuda_lib):
    """LSHSparseAttnServer(max_query_tokens=4) on a 3-layer config with generation_buffer = 16: a scripted speculative loop across
    spills.  Every accepted token's output equals (or is within one bf16 ulp of) a twin server that generates one at a time."""
    from magicpig_b200.attnserver import LSHSparseAttnServer
    cfg = _Cfg()
    K, L, B, P, M, gen = 8, 40, 2, 600, 1024, 16
    Hq, Hkv = cfg.num_attention_heads, cfg.num_key_value_heads
    hf = synth.make_hash_func(d, K, L, seed=41)
    g = torch.Generator().manual_seed(42)
    kc = [torch.randn((B, P, Hkv, d), generator=g).bfloat16() for _ in range(3)]
    vc = [torch.randn((B, P, Hkv, d), generator=g).bfloat16() for _ in range(3)]
    servers = []
    for mq in (4, 1):
        s = LSHSparseAttnServer(cfg, K=K, L=L, batch_size=B, generation_buffer=gen, max_length=M, dense_layers=(0,),
                                device=DEV, hash_func=hf.to(DEV), max_query_tokens=mq)
        s.alloc_buffer(P)
        for layer in range(3):
            for b in range(B):
                s.fill(layer, b, kc[layer][b].to(DEV), vc[layer][b].to(DEV), P)
                s.build_table(layer, b, P)
        servers.append(s)
    spec, twin = servers
    accepted_total, used = 0, 0
    for step, drop in enumerate([1, 0, 2, 3, 1, 0, 2, 1, 0, 3, 1, 2, 0, 1]):
        T = 4
        if used + T > gen:
            spec.spill_window()
            twin.spill_window()
            used = 0
        q = [torch.randn((B, Hq, T, d), generator=g).bfloat16().to(DEV) for _ in range(3)]
        k = [torch.randn((B, Hkv, T, d), generator=g).bfloat16().to(DEV) for _ in range(3)]
        v = [torch.randn((B, Hkv, T, d), generator=g).bfloat16().to(DEV) for _ in range(3)]
        spec.plan(T)
        outs = [spec.decode(q[l], k[l], v[l], l).clone() for l in range(3)]
        assert outs[1].shape == (B, T, Hq * d)
        spec.rewind(drop)
        for t in range(T - drop):
            twin.plan()
            for l in range(3):
                o = twin.decode(q[l][:, :, t:t + 1], k[l][:, :, t:t + 1], v[l][:, :, t:t + 1], l)
                # one bf16 ulp; near-zero elements (cancellation) against the row's scale instead
                a, b_ = outs[l][:, t].float(), o[:, 0].float()
                bound = torch.maximum(a.abs(), b_.abs()) * 2.0 ** -7 + 1e-5 * b_.abs().amax(dim=-1, keepdim=True)
                assert bool(((a - b_).abs() <= bound).all()), (step, l, t)
        used += T - drop
        accepted_total += T - drop
    assert accepted_total > 2 * gen
