"""GPU parity suite (`-m gpu`, runs on an H100 through the C ABI).

Every test drives the CUDA library (ctypes -> libmagicpig_b200.so) and checks it against the oracle
(oracle/mpig_oracle.c, pinned to the reference -- see tests/test_oracle_cpu.py) on the same seeded
inputs, against the committed golden vectors, and -- at BASELINE's full size -- through
size-independent properties.  Integer work (codes away from zero projections, index sets, nnz,
saturated and full collision counts) must match bit-exactly.  Floating point (BASELINE.json: "within 1e-3 relative on
the attention output"): the operator's output is bf16 by ABI (sparse_attention.cc:343-346), whose rounding alone is up to
2^-8 = 3.9e-3 of an element, so the 1e-3 bar is applied where it can be met by any implementation --
  * `assert_1e3_before_rounding`: |out - o| <= half-ulp_bf16(o) + 1e-3 * max|o| against the oracle's UN-rounded output
    o = sum_j p_j V_j (its fp32 probabilities, fp64 accumulation), i.e. 1e-3 on the arithmetic + the mandated rounding;
  * the fp32 base-2 LSE (the value the caller merges with) within 1e-3 absolute;
and, where both sides are already rounded to bf16 (oracle output, golden vectors of the compiled reference), one bf16
ulp: 4e-3 max-norm (6e-3 after the window merge, which rounds once more), the reference's own 1e-2 against its
compiled operators' golden outputs (they use a 3rd-order polynomial exp).
"""
import math
import os

import numpy as np
import pytest
import torch

import oracle
from magicpig_b200 import synth
from tests.support.fp64 import SIMHASH_EPS, assert_1e3_before_rounding, assert_1e3_f32, bf16_from_u16, oracle_decode
from tests.support.library import _Cfg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-12))


# ------------------------------------------------------------------------------------------------
# stage 2: probe  (mirrors library/lsh/test.py:5-76)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route", ["sorted", "device"])
@pytest.mark.parametrize("K,L,seq,delta,group,bsz,layers", [
    (4, 50, 1024, 128, 4, 1, 1), (8, 100, 4096, 1024, 8, 4, 2), (8, 50, 8192, 128, 4, 1, 2), (4, 100, 1024, 1024, 8, 4, 1),
    (2, 4, 128, 16, 1, 1, 1),
    # several 65536-key segments per table row (compact uint16 items): 3 segments (cluster padded to 4), and 2 segments
    # with 4 CTAs per segment
    (8, 20, 140000, 32, 4, 1, 1), (6, 12, 70000, 100, 1, 2, 1),
])
def test_batch_retrieve(cuda_lib, route, K, L, seq, delta, group, bsz, layers):
    from magicpig_b200.ops import LSH
    g = torch.Generator().manual_seed(K * 131 + L + seq)
    Hq = 32 if group > 1 else 1
    Hkv = Hq // group
    NB, M = 1 << K, seq + delta
    layer = layers - 1
    lsh = LSH(device=DEV)
    lsh.alloc(K, L, layers, Hq, Hkv, bsz, M)
    codes = torch.randint(0, NB, (bsz, Hkv, L, seq), generator=g, dtype=torch.int16)
    if route == "sorted":
        sc, si = codes.sort()
        for b in range(bsz):
            lsh.fill(layer, b, sc[b].to(DEV), si[b].int().to(DEV))
    else:
        for b in range(bsz):
            lsh.build(layer, b, codes[b].to(DEV))
    for rep in range(2):  # twice: scratch state must not leak between probes (test.py:59-75)
        query = torch.randint(0, NB, (bsz * Hq, L), generator=g, dtype=torch.int32)
        results = torch.zeros((bsz * Hq, M), dtype=torch.int32, device=DEV)
        nnz = torch.zeros((bsz * Hq,), dtype=torch.int32, device=DEV)
        lsh.batch_retrieve(layer, query.to(DEV), results, nnz)
        mask = lsh.get_mask().cpu().view(torch.uint8).reshape(bsz * Hq, M)
        counts_gpu = lsh.ctx.lsh_collision_counts(layer, query.to(DEV)).cpu()
        results, nnz = results.cpu(), nnz.cpu()
        for b in range(bsz):
            sl = slice(b * Hq, (b + 1) * Hq)
            cnt = oracle.collision_counts(codes[b].contiguous(), query[sl].contiguous(), group)
            assert torch.equal(nnz[sl], (cnt > 1).sum(-1).int())
            assert torch.equal(mask[sl, :seq], cnt.clamp(max=2).to(torch.uint8))       # get_mask(), lsh.cc:308-314
            assert int(mask[sl, seq:].sum()) == 0
            assert torch.equal(counts_gpu[sl, :seq], cnt)                               # full collision counts
            for h in range(Hq):
                got = results[b * Hq + h, : nnz[b * Hq + h]]
                want = torch.nonzero(cnt[h] > 1).flatten().int()
                assert torch.equal(got, want)  # ascending order == exact set


def test_probe_empty_and_ragged(cuda_lib):
    """n = 0 request, ragged n per request, query codes that miss everything."""
    from magicpig_b200.ops import LSH
    K, L, Hq, Hkv, B, M = 6, 24, 4, 2, 3, 300
    g = torch.Generator().manual_seed(1)
    lsh = LSH(device=DEV)
    lsh.alloc(K, L, 1, Hq, Hkv, B, M)
    ns = [0, 257, 300]
    codes = [torch.randint(0, 1 << K, (Hkv, L, n), generator=g, dtype=torch.int16) for n in ns]
    for b, c in enumerate(codes):
        lsh.build(0, b, c.to(DEV))
    query = torch.randint(0, 1 << K, (B * Hq, L), generator=g, dtype=torch.int32)
    results = torch.zeros((B * Hq, M), dtype=torch.int32, device=DEV)
    nnz = torch.zeros((B * Hq,), dtype=torch.int32, device=DEV)
    lsh.batch_retrieve(0, query.to(DEV), results, nnz)
    nnz, results = nnz.cpu(), results.cpu()
    assert int(nnz[:Hq].sum()) == 0
    for b in (1, 2):
        cnt = oracle.collision_counts(codes[b], query[b * Hq:(b + 1) * Hq].contiguous(), Hq // Hkv)
        assert torch.equal(nnz[b * Hq:(b + 1) * Hq], (cnt > 1).sum(-1).int())
    # clear() forgets every request (lsh.cc:293-306)
    lsh.clear()
    lsh.batch_retrieve(0, query.to(DEV), results.to(DEV), (nnz2 := torch.ones((B * Hq,), dtype=torch.int32, device=DEV)))
    assert int(nnz2.sum()) == 0


# ------------------------------------------------------------------------------------------------
# stage 3: gather attention  (mirrors library/sparse_attention/test_sparse.py:6-92)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seq,delta,group,bsz,Hq,tma", [(8192, 128, 4, 1, 32, 1), (8192, 1024, 8, 4, 32, 1), (2048, 128, 8, 1, 64, 1),
                                                        (300, 20, 4, 2, 8, 1), (2048, 128, 8, 1, 64, 0)])
def test_sparse_attention(cuda_lib, seq, delta, group, bsz, Hq, tma):
    from magicpig_b200.ops import SparseAttentionServer
    K, L, d, layers = 10, 150, 128, 2
    g = torch.Generator().manual_seed(seq + group + bsz)
    M, Hkv, layer = seq + delta, Hq // group, 1
    H = bsz * Hq
    key = torch.randn((bsz, Hkv, seq, d), generator=g).bfloat16()
    value = torch.randn((bsz, Hkv, seq, d), generator=g).bfloat16()
    key_norm = key.norm(p=2, dim=-1).float()
    query = torch.randn((bsz, Hq, 1, d), generator=g).bfloat16()
    query_norm = query.float().norm(p=2, dim=-1).reshape(H)
    nnz = torch.randint(1, seq, (H,), generator=g).int()
    nnz[0] = 1
    nnz[-1] = seq
    ind = torch.zeros((H, M), dtype=torch.int32)
    for i in range(H):
        ind[i, : nnz[i]] = torch.randperm(seq, generator=g)[: nnz[i]].int()
    srv = SparseAttentionServer(device=DEV)
    srv.alloc(layers, Hq, Hkv, d, bsz, M)
    srv.ctx.set_option("attend_tma", tma)
    srv.ctx.set_option("out_f32", 1)
    for b in range(bsz):
        srv.fill(layer, b, key[b].to(DEV), value[b].to(DEV), key_norm[b].to(DEV))
    out = torch.zeros((H, d), dtype=torch.bfloat16, device=DEV)
    mve = torch.zeros((2, H), dtype=torch.float32, device=DEV)
    srv.attention_wrapper(layer, K, L, out, mve, query.to(DEV), query_norm.to(DEV), ind.to(DEV), nnz.to(DEV))
    out, mve = out.cpu(), mve.cpu()
    out32 = srv.ctx.last_out_f32().cpu()
    # oracle (exact-math restatement of sparse_attention.cc)
    kp = torch.zeros((bsz * Hkv, M, d), dtype=torch.bfloat16)
    vp = torch.zeros((bsz * Hkv, M, d), dtype=torch.bfloat16)
    knp = torch.zeros((bsz * Hkv, M))
    kp[:, :seq], vp[:, :seq], knp[:, :seq] = key.reshape(-1, seq, d), value.reshape(-1, seq, d), key_norm.reshape(-1, seq)
    o_ref, mve_ref, score = oracle.attention_wrapper(kp, vp, knp, K, L, query.reshape(H, d), query_norm, ind, nnz, want_score=True)
    assert rel_err(out, o_ref) < 4e-3            # both sides round the output to bf16: one bf16 ulp
    # the 1e-3 bar, before the output rounding: the oracle's probabilities (fp32) times V, accumulated in fp64
    for i in range(H):
        sel = ind[i, : nnz[i]].long()
        if len(sel):
            o_pre = score[i, : nnz[i]].double() @ vp[i // group][sel].double()
            assert_1e3_before_rounding(out[i], o_pre)
            assert_1e3_f32(out32[i][None], o_pre[None])
    assert torch.allclose(mve[1], mve_ref[1], atol=1e-3), (mve[1] - mve_ref[1]).abs().max()
    # row 0 (max*log2e) hangs on ONE element's `1 - q^(L-1)(Lp+q)` fp32 cancellation (powf ulp differences between
    # CUDA and glibc are amplified near w ~ 1e-4); nothing consumes it (attnserver.py:302 reads row 1 only)
    assert torch.allclose(mve[0], mve_ref[0], atol=2e-2)
    # fp64 torch formula (test_sparse.py:68-84), tolerance 1e-3 relative on the un-rounded scale
    sets = [ind[i, : nnz[i]] for i in range(H)]
    o64, lse64 = synth.torch_reference_attention(key.reshape(-1, seq, d), value.reshape(-1, seq, d), key_norm.reshape(-1, seq),
                                                 query.reshape(H, d), sets, K, L, group)
    assert rel_err(out, o64) < 3e-3
    assert torch.allclose(mve[1].double(), lse64, atol=5e-3)  # fp64 formula vs the reference's fp32 expression order
    # the store reads back what was filled (get_key_cache / get_value_cache / get_key_norm)
    kc = srv.get_key_cache(layer).cpu()
    assert torch.equal(kc[:, :, :seq].view(torch.int16), key.view(torch.int16))
    assert torch.equal(srv.get_value_cache(layer).cpu()[:, :, :seq].view(torch.int16), value.view(torch.int16))
    assert torch.equal(srv.get_key_norm(layer).cpu()[:, :, :seq], key_norm)


@pytest.mark.parametrize("tma", [1, 0])
def test_sparse_attention_nnz0_and_tiny(cuda_lib, tma):
    """tma = 1: per-row cp.async.bulk copies (TMA engine, the default); tma = 0: per-row 16-byte cp.async copies (LSU path)."""
    from magicpig_b200.ops import SparseAttentionServer
    K, L, d, Hq, Hkv, B, n, M = 10, 150, 128, 8, 2, 1, 64, 96
    g = torch.Generator().manual_seed(4)
    key = torch.randn((B, Hkv, n, d), generator=g).bfloat16()
    value = torch.randn((B, Hkv, n, d), generator=g).bfloat16()
    kn = key.norm(p=2, dim=-1).float()
    q = torch.randn((Hq, d), generator=g).bfloat16()
    nnz = torch.tensor([0, 1, 2, 31, 32, 33, 0, 64], dtype=torch.int32)
    ind = torch.zeros((Hq, M), dtype=torch.int32)
    for i in range(Hq):
        ind[i, : nnz[i]] = torch.randperm(n, generator=g)[: nnz[i]].int()
    srv = SparseAttentionServer(device=DEV)
    srv.alloc(1, Hq, Hkv, d, B, M)
    srv.ctx.set_option("attend_tma", tma)
    srv.fill(0, 0, key[0].to(DEV), value[0].to(DEV), kn[0].to(DEV))
    out = torch.full((Hq, d), 7.0, dtype=torch.bfloat16, device=DEV)
    mve = torch.zeros((2, Hq), dtype=torch.float32, device=DEV)
    qn = q.float().norm(p=2, dim=-1)
    for _ in range(2):  # second launch reuses the self-resetting merge tickets
        srv.attention_wrapper(0, K, L, out, mve, q.to(DEV), qn.to(DEV), ind.to(DEV), nnz.to(DEV))
    out, mve = out.cpu(), mve.cpu()
    kp = torch.zeros((Hkv, M, d), dtype=torch.bfloat16); vp = torch.zeros((Hkv, M, d), dtype=torch.bfloat16); knp = torch.zeros((Hkv, M))
    kp[:, :n], vp[:, :n], knp[:, :n] = key[0], value[0], kn[0]
    o_ref, mve_ref, _ = oracle.attention_wrapper(kp, vp, knp, K, L, q, qn, ind, nnz)
    for h in (0, 6):  # nnz = 0: zeros and LSE = -inf (SURVEY 7.3 #7)
        assert float(out[h].float().abs().max()) == 0.0 and math.isinf(float(mve[1, h])) and float(mve[1, h]) < 0
    live = nnz > 0
    assert rel_err(out[live], o_ref[live]) < 4e-3
    assert torch.allclose(mve[1][live], mve_ref[1][live], atol=1e-3)


# ------------------------------------------------------------------------------------------------
# stage 1: SimHash
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,L,B,Hq", [(10, 150, 1, 32), (10, 150, 8, 32), (11, 300, 1, 32), (4, 50, 2, 8), (7, 13, 1, 1)])
def test_simhash(cuda_lib, K, L, B, Hq):
    from magicpig_b200.ops import Context
    d = 128
    ctx = Context(K, L, 1, Hq, Hq, d, B, 64, device=DEV)
    hf = synth.make_hash_func(d, K, L, seed=K + L)
    ctx.set_hash_func(hf.to(DEV))
    q = synth.make_query(B, Hq, d, seed=3)
    codes, qn = ctx.simhash(q.to(DEV))
    codes, qn = codes.cpu(), qn.cpu()
    ref, margin = oracle.simhash(q.reshape(-1, d), hf, K, L)
    bad = codes != ref
    # bit-exact except where a projection is within fp32 accumulation noise of zero (sign decided by summation order,
    # SURVEY 7.3 #3); no count allowance: every mismatch must be explained by its margin
    assert int(bad.sum()) == 0 or float(margin[bad].max()) < SIMHASH_EPS, (int(bad.sum()), float(margin[bad].max()))
    assert torch.allclose(qn, q.reshape(-1, d).float().norm(p=2, dim=-1), rtol=1e-6)


# ------------------------------------------------------------------------------------------------
# golden vectors produced by the reference's compiled operators (tests/golden/make_golden.py)
# ------------------------------------------------------------------------------------------------
def test_hashing_requires_projection(cuda_lib):
    """SimHash / key hash / decode before set_hash_func must fail loudly, not hash with a zero projection."""
    from magicpig_b200 import _native as N
    from magicpig_b200.ops import Context
    ctx = Context(6, 10, 1, 4, 2, 128, 1, 256, device=DEV)
    q = torch.zeros((4, 128), dtype=torch.bfloat16, device=DEV)
    with pytest.raises(N.MagicPigError):
        ctx.simhash(q)
    with pytest.raises(N.MagicPigError):
        ctx.hash_keys(torch.zeros((2, 100, 128), dtype=torch.bfloat16, device=DEV))
    ctx.set_hash_func(synth.make_hash_func(128, 6, 10, seed=0).to(DEV))
    ctx.simhash(q)


def _fused_vs_golden(ctx, q, H, d, gold_nnz, gold_results, gold_offsets, gold_out, staged_out):
    """The fused single-launch decode on the golden inputs, window empty (plan() never called, so it is exactly
    SimHash -> probe -> sampled attention): same nnz / index lists as the compiled reference, output within the reference's
    own tolerance of its golden output and within fp32 noise of the staged kernels' output."""
    ctx.set_option("save_mask", 1)
    ctx.set_option("out_f32", 1)
    Bkv = ctx.B * ctx.Hkv
    z0 = torch.zeros((Bkv, d), dtype=torch.bfloat16, device=DEV)
    out_f = ctx.decode(0, q.to(DEV), z0, z0)
    assert ctx.get_info("last_decode_fused") == 1
    nnz_f, res_f = ctx.last_probe(want_results=True)
    assert torch.equal(nnz_f.cpu(), gold_nnz)
    for h in range(H):
        lo, hi = (int(gold_offsets[h]), int(gold_offsets[h + 1])) if gold_offsets is not None else (0, int(gold_nnz[h]))
        assert torch.equal(res_f[h, : int(nnz_f[h])].cpu(), gold_results[lo:hi])
    out_f = out_f.cpu().reshape(H, d)
    assert torch.allclose(out_f.float(), gold_out.float(), rtol=1e-2, atol=1e-2)      # reference's own tolerance
    assert float((out_f.float() - staged_out.float()).abs().max()) <= 2 ** -7 * float(staged_out.float().abs().max())


def test_golden_small_chain(cuda_lib):
    from magicpig_b200.ops import Context
    z = np.load(os.path.join(GOLD, "small_chain.npz"))
    B, Hq, Hkv, d, K, L, n, M = [int(x) for x in z["dims"]]
    H = B * Hq
    ctx = Context(K, L, 1, Hq, Hkv, d, B, M, device=DEV)
    ctx.set_option("save_mask", 1)
    hf = bf16_from_u16(z["hash_func"]).reshape(d, K * L)
    ctx.set_hash_func(hf.to(DEV))
    key = bf16_from_u16(z["key"]).reshape(B, Hkv, n, d)
    value = bf16_from_u16(z["value"]).reshape(B, Hkv, n, d)
    kn = torch.from_numpy(z["key_norm"])
    kcodes = torch.from_numpy(z["kcodes"])
    q = bf16_from_u16(z["query"]).reshape(H, d)
    for b in range(B):
        ctx.attn_fill(0, b, key[b].to(DEV), value[b].to(DEV), kn[b].to(DEV))
        ctx.lsh_build(0, b, kcodes[b].to(DEV))
    codes, qn = ctx.simhash(q.to(DEV))
    assert torch.equal(codes.cpu(), torch.from_numpy(z["qcodes"]))
    results = torch.zeros((H, M), dtype=torch.int32, device=DEV)
    nnz = torch.zeros((H,), dtype=torch.int32, device=DEV)
    ctx.lsh_batch_retrieve(0, codes, results, nnz)
    assert torch.equal(nnz.cpu(), torch.from_numpy(z["nnz"]))
    assert torch.equal(ctx.lsh_get_mask().cpu().reshape(H, M), torch.from_numpy(z["mask"]))
    offs = z["results_offsets"]
    rs = torch.from_numpy(z["results_sorted"])
    for h in range(H):
        assert torch.equal(results[h, : int(nnz[h])].cpu(), rs[offs[h]:offs[h + 1]])
    out = torch.zeros((H, d), dtype=torch.bfloat16, device=DEV)
    mve = torch.zeros((2, H), dtype=torch.float32, device=DEV)
    ctx.attention_wrapper(0, K, L, out, mve, q.to(DEV), qn, results, nnz)
    ref_out = bf16_from_u16(z["out_bf16"]).reshape(H, d)
    assert torch.allclose(out.cpu().float(), ref_out.float(), rtol=1e-2, atol=1e-2)   # reference's own tolerance
    assert torch.allclose(mve.cpu()[1], torch.from_numpy(z["mve"])[1], atol=2e-2)
    _fused_vs_golden(ctx, q, H, d, torch.from_numpy(z["nnz"]), rs, offs, ref_out, out.cpu())
    # all-miss queries: nnz = 0 everywhere, zero output, LSE = -inf
    miss = torch.from_numpy(z["miss_qcodes"]).to(DEV)
    ctx.lsh_batch_retrieve(0, miss, results, nnz)
    assert int(nnz.sum()) == 0
    ctx.attention_wrapper(0, K, L, out, mve, q.to(DEV), qn, results, nnz)
    assert float(out.float().abs().max()) == 0.0 and bool(torch.isinf(mve[1]).all())


def test_golden_c1_chain(cuda_lib):
    """BASELINE config[0] (1 head, seq 4096, K10 L150) against the reference CPU path's outputs."""
    from magicpig_b200.ops import Context
    from tests.golden.make_golden import checksum
    z = np.load(os.path.join(GOLD, "c1_chain.npz"))
    B, Hq, Hkv, d, K, L, n, M = [int(x) for x in z["dims"]]
    hf = synth.make_hash_func(d, K, L, seed=0)
    q = synth.make_query(B, Hq, d, seed=1)
    key, value, kn, _ = synth.make_kv(B, Hkv, n, d, seed=2, dist="clustered", q_dirs=q.reshape(B, Hq, d)[:, :1].float())
    if checksum(hf, q, key, value, kn) != str(z["input_sha256"]):
        pytest.skip("torch RNG stream differs from the one that produced the fixture")
    ctx = Context(K, L, 1, Hq, Hkv, d, B, M, device=DEV)
    ctx.set_hash_func(hf.to(DEV))
    ctx.attn_fill(0, 0, key[0].to(DEV), value[0].to(DEV), kn[0].to(DEV))
    ctx.lsh_build(0, 0, synth.hash_keys(key, hf, K, L)[0].to(DEV))
    codes, qn = ctx.simhash(q.to(DEV))
    assert torch.equal(codes.cpu(), torch.from_numpy(z["qcodes"]))
    results = torch.zeros((1, M), dtype=torch.int32, device=DEV)
    nnz = torch.zeros((1,), dtype=torch.int32, device=DEV)
    ctx.lsh_batch_retrieve(0, codes, results, nnz)
    assert torch.equal(nnz.cpu(), torch.from_numpy(z["nnz"]))
    assert torch.equal(results[0, : int(nnz[0])].cpu(), torch.from_numpy(z["results_sorted"]))
    out = torch.zeros((1, d), dtype=torch.bfloat16, device=DEV)
    mve = torch.zeros((2, 1), dtype=torch.float32, device=DEV)
    ctx.attention_wrapper(0, K, L, out, mve, q.reshape(1, d).to(DEV), qn, results, nnz)
    ref_out = bf16_from_u16(z["out_bf16"]).reshape(1, d)
    assert torch.allclose(out.cpu().float(), ref_out.float(), rtol=1e-2, atol=1e-2)
    assert abs(float(mve[1, 0]) - float(z["mve"][1, 0])) < 2e-2
    _fused_vs_golden(ctx, q.reshape(1, d), 1, d, torch.from_numpy(z["nnz"]), torch.from_numpy(z["results_sorted"]), None, ref_out, out.cpu())


# ------------------------------------------------------------------------------------------------
# fused decode: SimHash -> probe -> attention over window + sample, vs the oracle chain + merge
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("B,Hq,Hkv,n,K,L,dist", [(1, 32, 8, 4096, 10, 150, "clustered"), (2, 8, 2, 1500, 8, 60, "gauss"), (1, 4, 4, 300, 6, 24, "gauss"),
                                                 (1, 8, 1, 70000, 8, 40, "clustered"), (4, 32, 8, 2000, 8, 60, "gauss"),
                                                 (5, 32, 8, 1200, 8, 40, "gauss"),
                                                 # more tables than a one-byte tag holds ids for: two and three tag passes (C4 is K11 L300)
                                                 (1, 8, 2, 3000, 11, 300, "gauss"), (1, 4, 1, 40000, 9, 520, "clustered"),
                                                 # edges: one table, a single offloaded key, odd head counts, 4096 buckets
                                                 (1, 6, 3, 17, 4, 1, "gauss"), (1, 2, 1, 1, 5, 3, "gauss"), (3, 12, 4, 999, 7, 33, "gauss"),
                                                 (2, 4, 4, 5000, 12, 20, "gauss"),
                                                 # 320 heads: more one-CTA-per-head CTAs than fit at once (several waves)
                                                 (10, 32, 8, 300, 6, 24, "gauss")])
def test_fused_decode(cuda_lib, B, Hq, Hkv, n, K, L, dist, impl):
    """mpig_decode -- impl 1: ONE fused launch per layer (fused.cu); impl 0: SimHash | probe | attend -- against the oracle chain.
    nnz bit-exact; the bf16 output within one bf16 ulp of the reference data flow; the fp32 output (before the ABI's rounding)
    within 1e-3 of the oracle's un-rounded result.  Shapes: cluster of 4 / 8 / 8 CTAs per head, two key segments (n = 70 000),
    128 heads with one CTA each (codes from the stand-alone SimHash kernel), and 160 heads (two 512-thread CTAs per SM)."""
    from magicpig_b200.ops import Context
    d, ns, nl, gen = 128, 4, 64, 8
    M = n + 256
    G = Hq // Hkv
    hf = synth.make_hash_func(d, K, L, seed=21)
    q = synth.make_query(B, Hq, d, seed=22)
    qd = q.reshape(B, Hkv, G, d)[:, :, 0].float()
    key, value, kn, avg = synth.make_kv(B, Hkv, n, d, seed=23, dist=dist, q_dirs=qd)
    g = torch.Generator().manual_seed(24)
    w = ns + nl
    win_k = torch.randn((B, Hkv, w, d), generator=g).bfloat16()
    win_v = torch.randn((B, Hkv, w, d), generator=g).bfloat16()
    kcodes = synth.hash_keys(key, hf, K, L)
    ctx = Context(K, L, 2, Hq, Hkv, d, B, M, ns, nl, gen, dense_layers=[0], device=DEV)
    ctx.set_option("decode_impl", impl)
    ctx.set_option("out_f32", 1)
    ctx.set_hash_func(hf.to(DEV))
    for b in range(B):
        ctx.attn_fill(1, b, key[b].to(DEV), value[b].to(DEV), kn[b].to(DEV))
        ctx.lsh_build(1, b, kcodes[b].to(DEV))
        ctx.window_fill(1, b, avg[b].reshape(Hkv, d).to(DEV), win_k[b].to(DEV), win_v[b].to(DEV))
    t = dict(B=B, Hq=Hq, Hkv=Hkv, d=d, K=K, L=L, n=n, M=M, hash_func=hf, kcodes=kcodes, key=key, value=value, key_norm=kn, avg_k=avg)
    wk_hist, wv_hist = win_k, win_v
    for step in range(3):
        k_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
        v_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
        qs = synth.make_query(B, Hq, d, seed=30 + step) if step else q
        ctx.plan()
        out = ctx.decode(1, qs.to(DEV), k_new.to(DEV), v_new.to(DEV)).cpu()
        assert ctx.get_info("last_decode_fused") == impl
        nnz_gpu, _ = ctx.last_probe()
        o32 = ctx.last_out_f32().cpu()
        o_ref, nz_ref, _, o_exact = oracle_decode(t, qs, k_new, v_new, wk_hist, wv_hist, G)
        assert torch.equal(nnz_gpu.cpu(), nz_ref)
        assert_1e3_f32(o32, o_exact)                                        # the 1e-3 bar, on the path the product runs
        assert_1e3_before_rounding(out.reshape(B * Hq, d), o_exact)         # and the bf16 output is that value, rounded once
        assert rel_err(out.reshape(B * Hq, d), o_ref) < 6e-3, step          # reference data flow (rounds twice)
        wk_hist = torch.cat([wk_hist, (k_new - avg)], dim=2)
        wv_hist = torch.cat([wv_hist, v_new], dim=2)
    # host-buffer entry point gives the same answer as the device-pointer one
    ctx.plan()
    k_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
    v_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
    out_h = torch.zeros((B, Hq * d), dtype=torch.bfloat16).pin_memory()
    ctx.decode_host(1, q.reshape(B * Hq, d).contiguous().pin_memory(), k_new.reshape(B * Hkv, d).contiguous().pin_memory(),
                    v_new.reshape(B * Hkv, d).contiguous().pin_memory(), out_h)
    o_ref, _, _, o_exact = oracle_decode(t, q, k_new, v_new, wk_hist, wv_hist, G)
    assert_1e3_before_rounding(out_h.reshape(B * Hq, d), o_exact)
    assert_1e3_f32(ctx.last_out_f32().cpu(), o_exact)
    # pageable (un-pinned) host buffers are accepted too: the call stages through its own pinned block
    out_p = torch.zeros((B, Hq * d), dtype=torch.bfloat16)
    wk_hist = torch.cat([wk_hist, (k_new - avg)], dim=2)
    wv_hist = torch.cat([wv_hist, v_new], dim=2)
    ctx.plan()
    ctx.decode_host(1, q.reshape(B * Hq, d).contiguous(), k_new.reshape(B * Hkv, d).contiguous(), v_new.reshape(B * Hkv, d).contiguous(), out_p)
    _, _, _, o_exact = oracle_decode(t, q, k_new, v_new, wk_hist, wv_hist, G)
    assert_1e3_before_rounding(out_p.reshape(B * Hq, d), o_exact)


def test_fused_decode_matches_three_launch_and_saves_probe(cuda_lib):
    """Same inputs through both decode variants: identical nnz, index lists, masks and codes (option "save_mask" makes the fused
    kernel write them out), fp32 outputs within 1e-5 of each other (same tile math, different partition of the rows), and the
    selected-key list is taken in several passes when it exceeds the shared-memory list ("fused_selcap")."""
    from magicpig_b200.ops import Context
    B, Hq, Hkv, n, K, L, d = 1, 8, 2, 3000, 6, 40, 128       # K = 6: ~9 % of the keys collide twice -> ~70 rows per CTA
    M, G = n + 200, Hq // Hkv
    hf = synth.make_hash_func(d, K, L, seed=5)
    q = synth.make_query(B, Hq, d, seed=6)
    key, value, kn, avg = synth.make_kv(B, Hkv, n, d, seed=7, dist="gauss")
    kcodes = synth.hash_keys(key, hf, K, L)
    g = torch.Generator().manual_seed(8)
    win_k = torch.randn((B, Hkv, 68, d), generator=g).bfloat16()
    win_v = torch.randn((B, Hkv, 68, d), generator=g).bfloat16()
    k_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
    v_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
    got = {}
    for name, impl, selcap in (("three", 0, 2048), ("fused", 1, 2048), ("fused_passes", 1, 16)):
        ctx = Context(K, L, 1, Hq, Hkv, d, B, M, device=DEV)
        ctx.set_option("decode_impl", impl)
        ctx.set_option("fused_selcap", selcap)
        ctx.set_option("save_mask", 1)
        ctx.set_option("out_f32", 1)
        ctx.set_hash_func(hf.to(DEV))
        ctx.attn_fill(0, 0, key[0].to(DEV), value[0].to(DEV), kn[0].to(DEV))
        ctx.lsh_build(0, 0, kcodes[0].to(DEV))
        ctx.window_fill(0, 0, avg[0].reshape(Hkv, d).to(DEV), win_k[0].to(DEV), win_v[0].to(DEV))
        ctx.plan()
        out = ctx.decode(0, q.to(DEV), k_new.to(DEV), v_new.to(DEV))
        nnz, res = ctx.last_probe(want_results=True)
        got[name] = dict(out=out.cpu(), o32=ctx.last_out_f32().cpu(), nnz=nnz.cpu(), res=res.cpu(), mask=ctx.lsh_get_mask().cpu())
        assert ctx.get_info("last_decode_fused") == impl
        del ctx
    ref = got["three"]
    assert int(ref["nnz"].max()) > 64, "test shape should give every CTA several tiles"
    cnt = oracle.collision_counts(kcodes[0].contiguous(), oracle.simhash(q.reshape(Hq, d), hf, K, L)[0], G)
    for name in ("fused", "fused_passes"):
        o = got[name]
        assert torch.equal(o["nnz"], ref["nnz"]) and torch.equal(o["nnz"], (cnt > 1).sum(-1).int())
        for h in range(Hq):
            assert torch.equal(o["res"][h, : o["nnz"][h]], ref["res"][h, : ref["nnz"][h]])
            assert torch.equal(o["res"][h, : o["nnz"][h]], torch.nonzero(cnt[h] > 1).flatten().int())
        assert torch.equal(o["mask"], ref["mask"])
        assert torch.equal(o["mask"].reshape(Hq, M)[:, :n], cnt.clamp(max=2).to(torch.uint8))
        assert float((o["o32"] - ref["o32"]).abs().max()) <= 1e-5 * float(ref["o32"].abs().max())


def test_window_overflow_is_reported(cuda_lib):
    """generation_buffer exhausted: mpig_plan refuses (MPIG_ESTATE) instead of silently overwriting the last window row, and
    the device-side flag is raised when the plan kernel itself saturates (what a replayed CUDA graph would hit)."""
    from magicpig_b200 import _native as N
    from magicpig_b200.ops import Context
    ctx = Context(6, 10, 1, 4, 2, 128, 1, 512, num_sink_tokens=2, num_local_tokens=2, generation_buffer=3, device=DEV)
    assert ctx.get_info("window_capacity") == 7
    ctx.window_fill(0, 0, torch.zeros((2, 128), dtype=torch.bfloat16, device=DEV), torch.zeros((2, 4, 128), dtype=torch.bfloat16, device=DEV),
                    torch.zeros((2, 4, 128), dtype=torch.bfloat16, device=DEV))
    for _ in range(3):
        ctx.plan()
    assert ctx.error_flags() == 0
    with pytest.raises(N.MagicPigError, match="window is full"):
        ctx.plan()
    assert ctx.error_flags() == 0          # refused on the host: the device state is untouched
    # the device-side check: capture plan() (the host mirror stops being exact) and replay past the capacity
    gph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(gph, stream=s):
            ctx.plan()
    gph.replay()
    torch.cuda.synchronize()
    assert ctx.error_flags() & 1
    ctx.clear()
    assert ctx.error_flags() == 0


@pytest.mark.parametrize("B,Hq,Hkv,P,impl", [(2, 8, 2, 777, 1), (1, 8, 1, 5000, 1), (3, 4, 4, 31, 1), (1, 32, 8, 20000, 1), (2, 8, 2, 777, 0)])
def test_dense_decode(cuda_lib, B, Hq, Hkv, P, impl):
    """Dense layers (attnserver.py:235-259): plain attention over the whole context + appended token.
    impl=1: GQA-shared dense kernel (every K|V record fetched once per kv-group); impl=0: generic gather kernel."""
    from magicpig_b200.ops import Context
    d = 128
    M = ((P + 300) // 256 + 1) * 256
    G = Hq // Hkv
    g = torch.Generator().manual_seed(5 + P)
    ctx = Context(4, 8, 1, Hq, Hkv, d, B, M, dense_layers=[0], alloc_dense_kv=True, device=DEV)
    ctx.set_option("dense_impl", impl)
    ctx.set_option("out_f32", 1)
    kc = torch.randn((B, P, Hkv, d), generator=g).bfloat16()
    vc = torch.randn((B, P, Hkv, d), generator=g).bfloat16()
    for b in range(B):
        ctx.dense_fill(0, b, kc[b].to(DEV), vc[b].to(DEV), P)
    kk, vv = kc.transpose(1, 2), vc.transpose(1, 2)
    for step in range(2):
        q = torch.randn((B, Hq, 1, d), generator=g).bfloat16() * (1.0 + step)
        k_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
        v_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
        ctx.plan()
        out = ctx.dense_decode(0, q.to(DEV), k_new.to(DEV), v_new.to(DEV)).cpu().reshape(B * Hq, d)
        kk = torch.cat([kk, k_new], dim=2)
        vv = torch.cat([vv, v_new], dim=2)
        o_ref, _ = oracle.window_attention(kk.reshape(B * Hkv, -1, d).contiguous(), vv.reshape(B * Hkv, -1, d).contiguous(),
                                           q.reshape(B * Hq, d), G)
        assert rel_err(out, o_ref) < 6e-3, (step, rel_err(out, o_ref))
        assert_1e3_f32(ctx.last_out_f32().cpu(), o_ref)                 # fp32 output vs the oracle's un-rounded fp32 result
        assert_1e3_before_rounding(out, o_ref)


def test_dense_decode_checks_out(cuda_lib):
    """A caller's `out` for dense_decode must be a contiguous bf16 tensor on the context's device with B*Hq*d elements: the
    kernels write B*Hq*d bf16 values through its pointer."""
    from magicpig_b200 import _native as N
    from magicpig_b200.ops import Context
    B, Hq, Hkv, d, P = 2, 8, 2, 128, 100
    g = torch.Generator().manual_seed(11)
    ctx = Context(4, 8, 1, Hq, Hkv, d, B, 512, dense_layers=[0], alloc_dense_kv=True, device=DEV)
    for b in range(B):
        ctx.dense_fill(0, b, torch.randn((P, Hkv, d), generator=g).bfloat16().to(DEV),
                       torch.randn((P, Hkv, d), generator=g).bfloat16().to(DEV), P)
    q = torch.randn((B, Hq, 1, d), generator=g).bfloat16().to(DEV)
    k = torch.randn((B, Hkv, 1, d), generator=g).bfloat16().to(DEV)
    v = torch.randn((B, Hkv, 1, d), generator=g).bfloat16().to(DEV)
    bad = [torch.empty((B, Hq * d), dtype=torch.float32, device=DEV),        # dtype
           torch.empty((B, Hq * d), dtype=torch.bfloat16),                    # device
           torch.empty((Hq * d, B), dtype=torch.bfloat16, device=DEV).t(),    # contiguity
           torch.empty((B, Hq * d // 2), dtype=torch.bfloat16, device=DEV)]   # size
    for out in bad:
        with pytest.raises(N.MagicPigError, match="^out: "):
            ctx.dense_decode(0, q, k, v, out)
    ctx.plan()
    good = torch.empty((B, Hq * d), dtype=torch.bfloat16, device=DEV)
    assert ctx.dense_decode(0, q, k, v, good) is good


# ------------------------------------------------------------------------------------------------
# the drop-in class on a small Llama-shaped config
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("table_build,key_hash", [("device", "tcgen05"), ("sorted", "torch"), ("sorted", "tcgen05")])
def test_attnserver_dropin(cuda_lib, table_build, key_hash):
    from magicpig_b200.attnserver import LSHSparseAttnServer
    cfg = _Cfg()
    K, L, B, P, M, d = 8, 40, 2, 600, 1024, 128
    Hq, Hkv = cfg.num_attention_heads, cfg.num_key_value_heads
    g = torch.Generator().manual_seed(6)
    hf = synth.make_hash_func(d, K, L, seed=2)
    srv = LSHSparseAttnServer(cfg, K=K, L=L, batch_size=B, max_length=M, generation_buffer=16, dense_layers=[0, 16],
                              device=DEV, hash_func=hf, table_build=table_build, key_hash=key_hash)
    kcs = [torch.randn((B, M, Hkv, d), generator=g).bfloat16() for _ in range(3)]
    vcs = [torch.randn((B, M, Hkv, d), generator=g).bfloat16() for _ in range(3)]
    srv.ctx.set_option("out_f32", 1)
    gpu_codes = []
    for b in range(B):
        srv.alloc_buffer(P)
        for layer in range(3):
            srv.fill(layer, b, kcs[layer][b].to(DEV), vcs[layer][b].to(DEV), P)
            srv.build_table(layer, b, P)   # (the reference calls it one layer late; order is equivalent per layer)
        gpu_codes.append(srv.hash_code_buffer[:, :, :P - 68].clone().cpu())   # the codes layer 2's tables were built from
    srv.plan()
    q = torch.randn((B, Hq, 1, d), generator=g).bfloat16()
    k_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
    v_new = torch.randn((B, Hkv, 1, d), generator=g).bfloat16()
    G = Hq // Hkv
    # dense layer 0
    o0 = srv.decode(q.to(DEV), k_new.to(DEV), v_new.to(DEV), 0).cpu()
    assert o0.shape == (B, 1, Hq * d)
    kk = torch.cat([kcs[0][:, :P].transpose(1, 2), k_new], dim=2).reshape(B * Hkv, P + 1, d)
    vv = torch.cat([vcs[0][:, :P].transpose(1, 2), v_new], dim=2).reshape(B * Hkv, P + 1, d)
    o_ref, _ = oracle.window_attention(kk, vv, q.reshape(B * Hq, d), G)
    assert rel_err(o0.reshape(B * Hq, d), o_ref) < 6e-3
    # sparse layer 2: rebuild the reference's view of fill() on the CPU and run the oracle chain
    layer = 2
    o2 = srv.decode(q.to(DEV), k_new.to(DEV), v_new.to(DEV), layer).cpu().reshape(B * Hq, d)
    o2_f32 = srv.ctx.last_out_f32().cpu()
    kc, vc = kcs[layer][:, :P], vcs[layer][:, :P]
    n = P - 68
    off_k = kc[:, 4:P - 64].transpose(1, 2).contiguous()
    off_v = vc[:, 4:P - 64].transpose(1, 2).contiguous()
    avg = off_k.mean(dim=2, keepdim=True)
    assert torch.allclose(avg.float(), srv.avg_k[layer].cpu().float(), atol=1e-2)
    avg = srv.avg_k[layer].cpu()  # GPU and CPU bf16 means can differ by an ulp; centre with the server's
    off_k = off_k - avg
    kn = off_k.norm(p=2, dim=-1).float()
    # what fill() stored is what the reference's fill() would store, up to the last bf16 digit of torch's CUDA vs CPU norm
    k_st, v_st, kn_st = (x.cpu() for x in srv.ctx.read_cache(layer))
    assert torch.equal(k_st[:, :, :n].view(torch.int16), off_k.view(torch.int16))
    assert torch.equal(v_st[:, :, :n].view(torch.int16), off_v.view(torch.int16))
    assert torch.allclose(kn_st[:, :, :n], kn, rtol=2 ** -7, atol=0)
    kcodes = torch.stack(gpu_codes)                                   # (B, Hkv, L, n) as hashed on the GPU
    ref_codes = synth.hash_keys(off_k, hf, K, L)
    assert int((kcodes != ref_codes).sum()) <= kcodes.numel() // 1000   # key-side hash parity proper: test_hash_keys_tcgen05
    win_k = torch.cat([kc[:, :4], kc[:, P - 64:P]], dim=1).transpose(1, 2) - avg
    win_v = torch.cat([vc[:, :4], vc[:, P - 64:P]], dim=1).transpose(1, 2)
    # oracle on EXACTLY the server's stored state (its key norms, its key codes): index set and nnz bit-exact, output at 1e-3
    t = dict(B=B, Hq=Hq, Hkv=Hkv, d=d, K=K, L=L, n=n, M=M, hash_func=hf, kcodes=kcodes, key=off_k, value=off_v,
             key_norm=kn_st[:, :, :n].contiguous(), avg_k=avg)
    o_ref, nz_ref, _, o_exact = oracle_decode(t, q, k_new, v_new, win_k, win_v, G)
    nnz_gpu, _ = srv.ctx.last_probe()
    assert torch.equal(nnz_gpu.cpu(), nz_ref)
    assert_1e3_f32(o2_f32, o_exact)
    assert_1e3_before_rounding(o2, o_exact)
    assert rel_err(o2, o_ref) < 6e-3
    srv.clear()


# ------------------------------------------------------------------------------------------------
# BASELINE full sizes: size-independent properties, one sparse layer each
#   C2 = config[1] Llama-3.1-8B B=1 P=98000 K10 L150; C3 = B=8 P=32768; C4 = the ProLong shape K11 L300 at its full
#   P=500000 (BASELINE's 32-layer C4 runs at P=200000 to fit 80 GB; one layer fits at 500K, the harder case for the tables)
#   C5 = Llama-3.1-70B under KV-head TP=8: the per-rank shape Hq 8, Hkv 1, n = 97 932 (attnserver_dist.py:252-254)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,P,K,L,Hq,Hkv", [("C2", 1, 98000, 10, 150, 32, 8), ("C3", 8, 32768, 10, 150, 32, 8),
                                                  ("C4", 1, 500000, 11, 300, 32, 8), ("C5rank", 1, 98000, 10, 150, 8, 1)])
def test_full_size_properties(cuda_lib, name, B, P, K, L, Hq, Hkv):
    from magicpig_b200.ops import Context
    d = 128
    M = ((P + 255) // 256) * 256 + 256
    n = P - 68
    G = Hq // Hkv
    H = B * Hq
    ctx = Context(K, L, 1, Hq, Hkv, d, B, M, device=DEV)
    if name in ("C2", "C5rank"):
        # every head's cluster resident at once: where the context needs no more key segments than that allows, the cluster
        # size is chosen so that one launch is ONE wave of clusters
        assert ctx.get_info("fused_cluster_waves") == 1
    ctx.set_option("save_mask", 1)
    g = torch.Generator(device=DEV).manual_seed(0)
    hf = torch.randn((d, K * L), generator=g, device=DEV).bfloat16()
    ctx.set_hash_func(hf)
    q = torch.randn((H, d), generator=g, device=DEV).bfloat16()
    keys, values, kns, kcs = [], [], [], []
    for b in range(B):
        key = torch.randn((Hkv, n, d), generator=g, device=DEV)
        qb = q[b * Hq:(b + 1) * Hq]
        key += 0.6 * qb.reshape(Hkv, G, d)[:, :1].float() * torch.rand((Hkv, n, 1), generator=g, device=DEV)  # some keys aligned with q
        key = key.bfloat16()
        key = key - key.mean(dim=1, keepdim=True)
        value = torch.randn((Hkv, n, d), generator=g, device=DEV).bfloat16()
        kn = key.norm(p=2, dim=-1).float()
        kcodes = ctx.hash_keys(key)                                    # tensor-core key-side SimHash at full size
        if name == "C2":                                               # ... equal to the reference-style torch glue
            ref_codes = synth.hash_keys(key, hf, K, L)
            bad = torch.nonzero(ref_codes != kcodes)                   # (g, l, key) triples, a few dozen of 117 M
            assert bad.shape[0] <= 4096
            if bad.shape[0]:   # each must have a projection within accumulation noise of zero (fp64 re-evaluation)
                kk = key[bad[:, 0], bad[:, 2]].double()                                         # (nb, d)
                cols = (bad[:, 1, None] * K + torch.arange(K, device=DEV)[None, :])              # (nb, K)
                hh = hf.double().t()[cols]                                                      # (nb, K, d)
                margin = (hh * kk[:, None, :]).sum(-1).abs().min(dim=-1).values
                assert float(margin.max()) < SIMHASH_EPS * float(key.float().norm(dim=-1).mean()), float(margin.max())
            del ref_codes
        ctx.attn_fill(0, b, key, value, kn)
        ctx.lsh_build(0, b, kcodes)
        keys.append(key); values.append(value); kns.append(kn); kcs.append(kcodes)
    codes, qn = ctx.simhash(q)
    results = torch.zeros((H, M), dtype=torch.int32, device=DEV)
    nnz = torch.zeros((H,), dtype=torch.int32, device=DEV)
    ctx.lsh_batch_retrieve(0, codes, results, nnz)
    # (1) selection rule against the torch formula on the GPU for every head (exact)
    cnt = torch.zeros((H, n), dtype=torch.int32, device=DEV)
    for b in range(B):
        kc = kcs[b].reshape(Hkv, 1, L, n).expand(Hkv, G, L, n).reshape(Hq, L, n)
        cb = codes[b * Hq:(b + 1) * Hq]
        for l0 in range(0, L, 10):
            cnt[b * Hq:(b + 1) * Hq] += (kc[:, l0:l0 + 10] == cb[:, l0:l0 + 10, None].to(torch.int16)).sum(dim=1).int()
    assert torch.equal(nnz, (cnt > 1).sum(-1).int())
    assert 0.002 < float(nnz.float().mean()) / n < 0.2
    mask = ctx.lsh_get_mask().reshape(H, M)
    assert torch.equal(mask[:, :n], cnt.clamp(max=2).to(torch.uint8))
    for h in range(H):
        r = results[h, : int(nnz[h])]
        assert bool((r[1:] > r[:-1]).all())                             # sortedness
        assert torch.equal(r, torch.nonzero(cnt[h] > 1).flatten().int())  # exact set
    del mask, cnt
    # (2) idempotence: probing again gives identical bytes
    results2 = torch.zeros_like(results); nnz2 = torch.zeros_like(nnz)
    ctx.lsh_batch_retrieve(0, codes, results2, nnz2)
    assert torch.equal(nnz, nnz2) and torch.equal(results, results2)
    # (3) sorted-route tables give the same sample as the device-built ones
    for b in range(B):
        sc, si = kcs[b].sort()
        ctx.lsh_fill(0, b, sc.contiguous(), si.int().contiguous())
        del sc, si
    ctx.lsh_batch_retrieve(0, codes, results2, nnz2)
    assert torch.equal(nnz, nnz2) and torch.equal(results, results2)
    # (4) attention: convex combination, LSE consistent with an fp32 torch evaluation on the GPU, linear in V
    out = torch.zeros((H, d), dtype=torch.bfloat16, device=DEV)
    mve = torch.zeros((2, H), dtype=torch.float32, device=DEV)
    ctx.attention_wrapper(0, K, L, out, mve, q, qn, results, nnz)
    for h in range(0, H, 5):
        b, hh = divmod(h, Hq)
        idx = results[h, : int(nnz[h])].long()
        kk, vv = keys[b][hh // G][idx].float(), values[b][hh // G][idx].float()
        s_ = kk @ q[h].float()
        cs = (s_ / (qn[h] * kns[b][hh // G][idx])).clamp(-1, 1)
        p = (1 - torch.arccos(cs.double()) / math.pi) ** K
        w = 1 - (1 - p) ** L - L * ((1 - p) ** (L - 1)) * p
        zz = s_.double() / math.sqrt(d) - torch.log(w + 1e-4)
        ref = torch.softmax(zz, 0) @ vv.double()
        assert rel_err(out[h], ref) < 4e-3
        assert abs(float(mve[1, h]) - float(torch.logsumexp(zz, 0) / math.log(2))) < 5e-3
    for b in range(B):
        ctx.attn_fill(0, b, keys[b], (2 * values[b].float()).bfloat16(), kns[b])       # V -> 2V  => o -> 2o
    out2 = torch.zeros_like(out)
    ctx.attention_wrapper(0, K, L, out2, mve, q, qn, results, nnz)
    assert rel_err(out2.float(), 2 * out.float()) < 8e-3


# ------------------------------------------------------------------------------------------------
# harness-side fused elementwise kernels (include/magicpig_b200_aux.h) and the decode harness itself
# ------------------------------------------------------------------------------------------------
def test_aux_ops(cuda_lib):
    import ctypes
    from magicpig_b200 import _native as N
    import torch.nn.functional as F
    lib = N.load()
    g = torch.Generator(device=DEV).manual_seed(0)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rows, hs = 3, 4096
    h = torch.randn((rows, hs), generator=g, device=DEV).bfloat16()
    dl = torch.randn((rows, hs), generator=g, device=DEV).bfloat16()
    w = torch.randn((hs,), generator=g, device=DEV).bfloat16()
    h2, x = h.clone(), torch.empty_like(h)
    N.check(lib.mpig_aux_add_rmsnorm(P(h2), P(dl), P(w), 1e-5, P(x), rows, hs, st))
    href = h + dl
    xref = F.rms_norm(href.float(), (hs,), w.float(), 1e-5)
    assert torch.equal(h2, href)
    assert torch.allclose(x.float(), xref, rtol=2e-2, atol=2e-2)
    B, Hq, Hkv, d = 2, 8, 2, 128
    qkv = torch.randn((B, (Hq + 2 * Hkv) * d), generator=g, device=DEV).bfloat16()
    cos = torch.randn((64, d), generator=g, device=DEV).bfloat16()
    sin = torch.randn((64, d), generator=g, device=DEV).bfloat16()
    pos = torch.tensor([5, 17], device=DEV, dtype=torch.long)
    q = torch.empty((B, Hq, d), dtype=torch.bfloat16, device=DEV); k = torch.empty((B, Hkv, d), dtype=torch.bfloat16, device=DEV)
    v = torch.empty_like(k)
    N.check(lib.mpig_aux_rope_split(P(qkv), P(cos), P(sin), P(pos), P(q), P(k), P(v), B, Hq, Hkv, st))
    heads = qkv.reshape(B, Hq + 2 * Hkv, d).float()
    c, s = cos[pos][:, None].float(), sin[pos][:, None].float()
    rot = lambda t: torch.cat([-t[..., 64:], t[..., :64]], dim=-1)  # noqa: E731
    ref = heads * c + rot(heads) * s
    assert torch.allclose(q.float(), ref[:, :Hq], rtol=2e-2, atol=2e-2)
    assert torch.allclose(k.float(), ref[:, Hq:Hq + Hkv], rtol=2e-2, atol=2e-2)
    assert torch.equal(v, qkv.reshape(B, Hq + 2 * Hkv, d)[:, Hq + Hkv:])
    it = 1024
    gu = torch.randn((rows, 2 * it), generator=g, device=DEV).bfloat16()
    o = torch.empty((rows, it), dtype=torch.bfloat16, device=DEV)
    N.check(lib.mpig_aux_silu_mul(P(gu), P(o), rows, it, st))
    assert torch.allclose(o.float(), F.silu(gu[:, :it].float()) * gu[:, it:].float(), rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("rows,N_out,K_in", [(1, 4096, 4096), (1, 6144, 4096), (3, 1000, 512), (8, 130, 256), (1, 4096, 14336), (7, 33, 14336)])
def test_aux_gemv(cuda_lib, rows, N_out, K_in):
    """decode-batch linear layer as a weight-streaming GEMV, plain and with the fused SwiGLU epilogue."""
    import ctypes
    from magicpig_b200 import _native as N
    import torch.nn.functional as F
    lib = N.load()
    g = torch.Generator(device=DEV).manual_seed(rows * 7 + N_out)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    x = torch.randn((rows, K_in), generator=g, device=DEV).bfloat16()
    w = (torch.randn((N_out, K_in), generator=g, device=DEV) * 0.05).bfloat16()
    y = torch.empty((rows, N_out), dtype=torch.bfloat16, device=DEV)
    N.check(lib.mpig_aux_gemv(P(w), P(x), P(y), rows, N_out, K_in, 0, st))
    ref = x.double() @ w.double().t()
    scale = float(ref.abs().max())
    assert float((y.double() - ref).abs().max()) < 1e-2 * scale        # one bf16 rounding of an fp32 sum
    assert float((y.double() - F.linear(x, w).double()).abs().max()) < 1.6e-2 * scale
    if N_out % 2 == 0:
        half = N_out // 2                                                  # w = [gate; up]
        y2 = torch.empty((rows, half), dtype=torch.bfloat16, device=DEV)
        N.check(lib.mpig_aux_gemv(P(w), P(x), P(y2), rows, half, K_in, 1, st))
        gu = F.linear(x, w)
        ref2 = F.silu(gu[:, :half].float()) * gu[:, half:].float()
        assert float((y2.float() - ref2).abs().max()) < 2e-2 * float(ref2.abs().max()) + 1e-3
    with pytest.raises(N.MagicPigError):
        N.check(lib.mpig_aux_gemv(P(w), P(x), P(y), 9, N_out, K_in, 0, st))


@pytest.mark.parametrize("rows,Hq,Hkv,hs,inter", [(1, 32, 8, 4096, 14336), (3, 4, 2, 512, 1024), (8, 8, 1, 1024, 768)])
def test_aux_fused_linear(cuda_lib, rows, Hq, Hkv, hs, inter):
    """norm+qkv+rope and norm+gate/up+swiglu kernels against the unfused chain add_rmsnorm -> gemv -> rope_split / silu_mul."""
    import ctypes
    from magicpig_b200 import _native as N
    lib = N.load()
    g = torch.Generator(device=DEV).manual_seed(hs + rows)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    d = 128
    nq = (Hq + 2 * Hkv) * d
    h = torch.randn((rows, hs), generator=g, device=DEV).bfloat16()
    dl = torch.randn((rows, hs), generator=g, device=DEV).bfloat16()
    lnw = (1 + 0.1 * torch.randn((hs,), generator=g, device=DEV)).bfloat16()
    wqkv = (torch.randn((nq, hs), generator=g, device=DEV) * 0.03).bfloat16()
    wgu = (torch.randn((2 * inter, hs), generator=g, device=DEV) * 0.03).bfloat16()
    cos = torch.randn((64, d), generator=g, device=DEV).bfloat16()
    sin = torch.randn((64, d), generator=g, device=DEV).bfloat16()
    pos = torch.randint(0, 64, (rows,), generator=g, device=DEV, dtype=torch.long)
    for delta in (dl, None):
        # unfused chain
        h_ref, x_ref = h.clone(), torch.empty_like(h)
        N.check(lib.mpig_aux_add_rmsnorm(P(h_ref), P(delta) if delta is not None else None, P(lnw), 1e-5, P(x_ref), rows, hs, st))
        qkv = torch.empty((rows, nq), dtype=torch.bfloat16, device=DEV)
        N.check(lib.mpig_aux_gemv(P(wqkv), P(x_ref), P(qkv), rows, nq, hs, 0, st))
        q_r = torch.empty((rows, Hq, d), dtype=torch.bfloat16, device=DEV); k_r = torch.empty((rows, Hkv, d), dtype=torch.bfloat16, device=DEV)
        v_r = torch.empty_like(k_r)
        N.check(lib.mpig_aux_rope_split(P(qkv), P(cos), P(sin), P(pos), P(q_r), P(k_r), P(v_r), rows, Hq, Hkv, st))
        act_r = torch.empty((rows, inter), dtype=torch.bfloat16, device=DEV)
        N.check(lib.mpig_aux_gemv(P(wgu), P(x_ref), P(act_r), rows, inter, hs, 1, st))
        # fused
        h_out = torch.zeros_like(h)
        q = torch.zeros_like(q_r); k = torch.zeros_like(k_r); v = torch.zeros_like(v_r)
        N.check(lib.mpig_aux_norm_qkv_rope(P(wqkv), P(h), P(delta) if delta is not None else None, P(lnw), 1e-5, P(h_out), P(cos), P(sin),
                                           P(pos), P(q), P(k), P(v), rows, Hq, Hkv, hs, st))
        assert torch.equal(h_out, h_ref)                       # the residual stream is bit-identical
        for got, want in ((q, q_r), (k, k_r), (v, v_r)):
            assert float((got.float() - want.float()).abs().max()) <= 2e-2 * float(want.float().abs().max())
        act = torch.zeros_like(act_r)
        h_out2 = torch.zeros_like(h)
        N.check(lib.mpig_aux_norm_gemv(P(wgu), P(h), P(delta) if delta is not None else None, P(lnw), 1e-5, P(h_out2), P(act), rows, inter, hs, 1, st))
        assert torch.equal(h_out2, h_ref)
        assert float((act.float() - act_r.float()).abs().max()) <= 2e-2 * float(act_r.float().abs().max()) + 1e-3
    with pytest.raises(N.MagicPigError):   # in-place residual update is refused (every CTA re-reads h_in)
        N.check(lib.mpig_aux_norm_gemv(P(wgu), P(h), None, P(lnw), 1e-5, P(h), P(act), rows, inter, hs, 1, st))


def test_runner_fused_matches_eager_and_graph(cuda_lib):
    from magicpig_b200.llama_runner import LlamaDecodeRunner, LlamaShape
    shape = LlamaShape("tiny", 3, 512, 1024, 4, 2, 1000, 500000.0, 1e-5)
    # (1) fused glue == eager glue.  All layers dense here: LSH sampling is discrete, so bf16-level differences in q
    #     between the two code paths would legitimately change the sampled set of a sparse layer.
    outs = []
    for fused in (False, True):
        r = LlamaDecodeRunner(shape, 8, 40, 2, 1024, device=DEV, seed=3, generation_buffer=16, dense_layers=(0, 1, 2), fused=fused)
        r.synthetic_prefill(600, seed=9)
        r.ids.fill_(7)
        outs.append([r.step().clone() for _ in range(2)])
        del r
    for a, b in zip(outs[0], outs[1]):
        assert torch.allclose(a, b, rtol=5e-2, atol=5e-2), float((a - b).abs().max())
    # (2) sparse layers under CUDA-graph capture/replay: finite logits, window advances, replay is repeatable in shape
    r = LlamaDecodeRunner(shape, 8, 40, 2, 1024, device=DEV, seed=3, generation_buffer=16, dense_layers=(0,), fused=True)
    r.synthetic_prefill(600, seed=9)
    r.ids.fill_(7)
    eager = r.step().clone()
    r.capture(warm=1)
    rep = r.replay().clone()
    assert torch.isfinite(eager).all() and torch.isfinite(rep).all()
    assert float(rep.abs().max()) < 50 * float(eager.abs().max()) + 1.0  # same model, next position: same scale
    nnz, _ = r.server.ctx.last_probe()
    assert int(nnz.sum()) > 0


# ------------------------------------------------------------------------------------------------
# key-side SimHash on the tensor cores (table build, SURVEY 8(f)-1): mirrors attnserver.py:159-168
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("K,L,Hkv,n", [(10, 150, 2, 1000), (11, 300, 1, 777), (4, 50, 8, 128), (15, 16, 1, 4097), (7, 13, 3, 130),
                                       (10, 150, 8, 20011), (1, 3, 1, 5)])
def test_hash_keys_tcgen05(cuda_lib, K, L, Hkv, n, impl):
    from magicpig_b200.ops import Context
    d = 128
    ctx = Context(K, L, 1, Hkv, Hkv, d, 1, max(n, 64) + 64, device=DEV)
    hf = synth.make_hash_func(d, K, L, seed=K * L)
    ctx.set_hash_func(hf.to(DEV))
    ctx.set_option("keyhash_impl", impl)   # 1 = persistent warp-specialised pipeline, 0 = one tile per CTA
    g = torch.Generator().manual_seed(n)
    keys = torch.randn((Hkv, n, d), generator=g).bfloat16()
    keys[:, n // 2] = 0                     # an all-zero key hashes to code 0 in every table (gt(0) is strict)
    codes = ctx.hash_keys(keys.to(DEV)).cpu()                       # (Hkv, L, n) int16
    proj = (keys.double().reshape(-1, d) @ hf.double()).reshape(Hkv, n, L, K)   # exact products, fp64 sums
    ref_bits = (proj > 0)
    ref = (ref_bits.long() * (2 ** torch.arange(K))).sum(-1).permute(0, 2, 1).to(torch.int16)   # (Hkv, L, n)
    bad = codes != ref
    if bad.any():
        # a code may differ only where one of its K projections is within fp32 accumulation noise of zero; the projections of
        # un-normalised N(0,1) keys have standard deviation sqrt(d).  No count allowance.
        margin = proj.abs().min(dim=-1).values.permute(0, 2, 1)    # (Hkv, L, n)
        assert float(margin[bad].max()) < SIMHASH_EPS * math.sqrt(d), (int(bad.sum()), float(margin[bad].max()))
    assert int(codes[:, :, n // 2].abs().sum()) == 0
    # and it feeds the table build: same tables as from the reference-style hash
    ctx.lsh_build(0, 0, codes.to(DEV))


# ------------------------------------------------------------------------------------------------
# accuracy-harness stand-in (SURVEY 8 f4): the "Masked" torch formulation the reference evaluates RULER with
# (evaluations/RULER/pred/attnserver_dist.py:813-851) against the GPU decode, several steps at the full C2 size
# ------------------------------------------------------------------------------------------------
def masked_formulation(q, keys, values, kn, kcodes, qcodes, K, L, G):
    """attnserver_dist.py:813-851 restated in fp32/fp64 torch on the GPU for ONE request: mask = #collisions > 1
    (:820-822), scores q.K^T, cos -> theta -> weight (:835-841), s/sqrt(d) - log(w + 1e-4) (:845-846), masked softmax and base-2
    LSE (:848-851).  The reference formulation rounds the scores and the probabilities to bf16 (its tensors are bf16); this
    restatement keeps fp32 scores like the CPU operator it stands in for (sparse_attention.cc:38-67).
    q (Hq, d) bf16; keys/values (Hkv, n, d) bf16; kn (Hkv, n) fp32; kcodes (Hkv, L, n) int16; qcodes (Hq, L) int32.
    Returns out (Hq, d) fp64, lse2 (Hq,) fp64, mask (Hq, n) bool."""
    Hq, d = q.shape
    Hkv, n, _ = keys.shape
    mask = torch.zeros((Hq, n), dtype=torch.int32, device=q.device)
    kc = kcodes.reshape(Hkv, 1, L, n).expand(Hkv, G, L, n).reshape(Hq, L, n)
    for l0 in range(0, L, 10):
        mask += (kc[:, l0:l0 + 10] == qcodes[:, l0:l0 + 10, None].to(torch.int16)).sum(dim=1).int()
    mask = mask > 1
    kk = keys.reshape(Hkv, 1, n, d).expand(Hkv, G, n, d).reshape(Hq, n, d)
    s = torch.einsum("hnd,hd->hn", kk.float(), q.float())                       # exact bf16 products, fp32 sums
    knn = kn.reshape(Hkv, 1, n).expand(Hkv, G, n).reshape(Hq, n)
    qn = q.float().norm(p=2, dim=-1, keepdim=True)
    cs = (s / (knn * qn)).clamp(-1, 1).double()
    w = 1 - torch.arccos(cs) / math.pi
    w = 1 - (1 - w ** K) ** L - L * ((1 - w ** K) ** (L - 1)) * (w ** K)
    z = s.double() / math.sqrt(d) - torch.log(w + 1e-4)
    z = z.masked_fill(~mask, -math.inf)
    lse2 = torch.logsumexp(z, dim=-1) / math.log(2)
    p = torch.softmax(z, dim=-1)
    p = torch.where(mask.any(dim=-1, keepdim=True), p, torch.zeros_like(p))
    vv = values.reshape(Hkv, 1, n, d).expand(Hkv, G, n, d).reshape(Hq, n, d)
    out = torch.einsum("hn,hnd->hd", p, vv.double())
    return out, lse2, mask


def test_masked_formulation_c2_steps(cuda_lib):
    """8 decode steps at the C2 size (Llama-3.1-8B head shape, n = 97 932, K10 L150) on clustered (heavy-tailed) keys: per
    step the GPU decode's sampled set is exactly the Masked formulation's mask (workload/decode_tokens of
    attnserver_dist.py:824-825 == mean nnz/n), and its fp32 output is within 1e-3 of mask-attention merged with the window."""
    from magicpig_b200.ops import Context
    B, Hq, Hkv, d, K, L, P = 1, 32, 8, 128, 10, 150, 98000
    n, M, G = P - 68, 98304, 4
    ctx = Context(K, L, 1, Hq, Hkv, d, B, M, device=DEV)
    ctx.set_option("save_mask", 1)
    ctx.set_option("out_f32", 1)
    g = torch.Generator(device=DEV).manual_seed(42)
    hf = torch.randn((d, K * L), generator=g, device=DEV).bfloat16()
    ctx.set_hash_func(hf)
    # clustered keys: 8 directions per kv-head, exponential strengths -> a heavy tail of keys aligned with each other
    centres = torch.randn((Hkv, 8, d), generator=g, device=DEV)
    assign = torch.randint(0, 8, (Hkv, n), generator=g, device=DEV)
    strength = -torch.log(torch.rand((Hkv, n, 1), generator=g, device=DEV)) * 0.7
    key = torch.randn((Hkv, n, d), generator=g, device=DEV) + strength * torch.gather(centres, 1, assign[..., None].expand(Hkv, n, d))
    key = key.bfloat16()
    avg = key.float().mean(dim=1, keepdim=True).bfloat16()
    key = key - avg
    value = torch.randn((Hkv, n, d), generator=g, device=DEV).bfloat16()
    kn = key.norm(p=2, dim=-1).float()
    kcodes = ctx.hash_keys(key)
    ctx.attn_fill(0, 0, key, value, kn)
    ctx.lsh_build(0, 0, kcodes)
    win_k = torch.randn((Hkv, 68, d), generator=g, device=DEV).bfloat16()
    win_v = torch.randn((Hkv, 68, d), generator=g, device=DEV).bfloat16()
    ctx.window_fill(0, 0, avg.reshape(Hkv, d), win_k, win_v)
    wk, wv = win_k, win_v
    workload = 0.0
    for step in range(8):
        # queries near one of the key clusters, like a decode query attending to its topic
        qd = centres[:, step % 8].reshape(Hkv, 1, d) + 0.8 * torch.randn((Hkv, G, d), generator=g, device=DEV)
        q = (qd.reshape(Hq, d) * 1.5).bfloat16()
        k_new = torch.randn((Hkv, d), generator=g, device=DEV).bfloat16()
        v_new = torch.randn((Hkv, d), generator=g, device=DEV).bfloat16()
        ctx.plan()
        out = ctx.decode(0, q, k_new, v_new)
        assert ctx.get_info("last_decode_fused") == 1
        nnz, res = ctx.last_probe(want_results=True)
        codes = ctx.last_codes()
        o32 = ctx.last_out_f32()
        # the fused kernel's own hash against the formulation's (torch bf16 GEMM, :815-819): equal except within noise of zero
        nq = (q / q.norm(p=2, dim=-1, keepdim=True))
        proj = nq.double() @ hf.double()
        ref_codes = ((proj > 0).reshape(Hq, L, K).long() * (2 ** torch.arange(K, device=DEV))).sum(-1).int()
        bad = codes != ref_codes
        if bad.any():
            margin = proj.abs().reshape(Hq, L, K).min(dim=-1).values
            assert float(margin[bad].max()) < SIMHASH_EPS
        o_m, lse_m, mask = masked_formulation(q, key, value, kn, kcodes, codes, K, L, G)
        assert torch.equal(nnz, mask.sum(-1).int())
        for h in range(0, Hq, 7):
            assert torch.equal(res[h, : int(nnz[h])].long(), torch.nonzero(mask[h]).flatten())
        workload += float(mask.float().mean())
        # window state (sink + local + generated rows incl. this token) and the LSE merge (:853-881), fp64
        wk = torch.cat([wk, (k_new - avg.reshape(Hkv, d)).reshape(Hkv, 1, d)], dim=1)
        wv = torch.cat([wv, v_new.reshape(Hkv, 1, d)], dim=1)
        wkk = wk.reshape(Hkv, 1, -1, d).expand(Hkv, G, wk.shape[1], d).reshape(Hq, -1, d)
        wvv = wv.reshape(Hkv, 1, -1, d).expand(Hkv, G, wv.shape[1], d).reshape(Hq, -1, d)
        zw = torch.einsum("hnd,hd->hn", wkk.float(), q.float()).double() / math.sqrt(d)
        lse_w = torch.logsumexp(zw, dim=-1) / math.log(2)
        o_w = torch.einsum("hn,hnd->hd", torch.softmax(zw, dim=-1), wvv.double())
        mx = torch.maximum(lse_w, lse_m)
        a, b_ = torch.exp2(lse_w - mx), torch.exp2(lse_m - mx)
        o_exact = (a[:, None] * o_w + b_[:, None] * o_m) / (a + b_)[:, None]
        assert_1e3_f32(o32, o_exact)
        assert_1e3_before_rounding(out.reshape(Hq, d), o_exact)
    workload /= 8
    assert 0.002 < workload < 0.2, workload      # README.md:43: ~2 % of the keys are attended at K10 L150
