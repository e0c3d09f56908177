"""Prefill attention (mpig_prefill_attend, csrc/attend_prefill.cu) against fp64, and LlamaDecodeRunner.prefill end to end.

Every case first shows that the named perturbations of tests/support/prefill_cases.py (causal limit +-1, top-left alignment, kv-head
h mod Hkv, the last key tile dropped, one tile's rescale skipped) move the fp64 output by >= 10x the bar; then the fp32 output is
within 1e-3 of each row's max-norm of fp64 and the bf16 output is the fp32 output rounded half-up, element for element."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from magicpig_b200 import _native as N
from tests.support.fp64 import assert_1e3_f32, assert_rounded_half_up
from tests.support.prefill_cases import REGIMES, Case, check_rows

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
d, K_, L_ = 128, 6, 16
_CTX = {}


def ctx_for(Hq, Hkv):
    from magicpig_b200.ops import Context
    if (Hq, Hkv) not in _CTX:
        _CTX[(Hq, Hkv)] = Context(K_, L_, 1, Hq, Hkv, d, 1, 1024, device=DEV)
    return _CTX[(Hq, Hkv)]


def run_case(c, tokens=None, probe=None):
    """Check the inputs, run the kernel once and compare the rows `tokens` (None: all) with fp64."""
    o64, _ = c.check_inputs(tokens, probe)
    ctx = ctx_for(c.Hq, c.Hkv)
    out = torch.full((c.q_len, c.Hq, d), float("nan"), dtype=torch.bfloat16, device=DEV)
    f32 = torch.full((c.q_len, c.Hq, d), float("nan"), dtype=torch.float32, device=DEV)
    ctx.prefill_attend(c.q, c.k, c.v, out, f32)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(f32).all()), "rows left unwritten or not finite"
    sel = slice(None) if tokens is None else tokens.to(DEV)
    assert_1e3_f32(f32[sel], o64)
    assert_rounded_half_up(out[sel], f32[sel])
    return out, f32


SMALL = [(1, 1), (1, 5), (7, 7), (64, 129), (129, 129), (300, 1000),
         # one off a tile edge on both axes: 32 tokens per m-block at G = 4, 128 keys per tile
         (31, 127), (33, 129), (32, 128), (31, 255), (33, 257), (95, 1023), (97, 1025)]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("q_len,kv_len", SMALL)
def test_small_and_ragged(q_len, kv_len, regime):
    run_case(Case(regime, q_len, kv_len, 32, 8, seed=q_len * 7 + kv_len))


# G in {1, 4, 7, 8}: 18 tokens per m-block at G = 7, the 70B per-rank shape Hq 8 / Hkv 1 at G = 8
GQA = [(8, 8, 1000, 1500), (32, 8, 1000, 1500), (28, 4, 700, 1201), (8, 1, 600, 1000), (64, 8, 300, 700)]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("Hq,Hkv,q_len,kv_len", GQA)
def test_gqa_groups(Hq, Hkv, q_len, kv_len, regime):
    run_case(Case(regime, q_len, kv_len, Hq, Hkv, seed=Hq + Hkv))


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("q_len,kv_len", [(8192, 8192), (7888, 98000)])
def test_llama8b_chunks(q_len, kv_len, regime):
    """A reference chunk of 8 192 tokens, and the last chunk of a 98 000-token prompt: every row checked."""
    c = Case(regime, q_len, kv_len, 32, 8, seed=11)
    run_case(c, None, check_rows(q_len, c.G, n_random=128))


@pytest.mark.parametrize("regime", REGIMES)
def test_whole_98k_prompt(regime):
    """(98 000, 98 000) in one call: first and last rows, each m-block's first and last row and 1 024 random rows."""
    c = Case(regime, 98000, 98000, 32, 8, seed=13)
    rows = check_rows(98000, c.G, n_random=1024)
    probe = check_rows(98000, c.G, n_random=64)
    run_case(c, rows, torch.cat([probe[:-1:16], probe[-1:]]))   # every 16th, and the last row


def test_capture_replays_bitwise():
    c = Case("sinks", 1000, 3000, 32, 8, seed=17)
    ctx = ctx_for(32, 8)
    eager = ctx.prefill_attend(c.q, c.k, c.v)
    out = torch.zeros_like(eager)
    f32 = torch.zeros(out.shape, dtype=torch.float32, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ctx.prefill_attend(c.q, c.k, c.v, out, f32)   # warm-up (function attributes, tensor-map encoder)
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ctx.prefill_attend(c.q, c.k, c.v, out, f32)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), eager.view(torch.int16))
    assert_rounded_half_up(out, f32)


def test_refusals():
    """Lengths, null and misaligned pointers: MPIG_EINVAL before anything is launched; the Python front-end refuses bad tensors."""
    ctx = ctx_for(32, 8)
    q = torch.zeros((8, 32, d), dtype=torch.bfloat16, device=DEV)
    k = torch.zeros((16, 8, d), dtype=torch.bfloat16, device=DEV)
    out = torch.empty_like(q)
    f32 = torch.empty(q.shape, dtype=torch.float32, device=DEV)
    P = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)   # noqa: E731
    NUL = ctypes.c_void_p(0)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = ctx.lib.mpig_prefill_attend
    EINVAL = -1
    assert call(ctx._h, P(q), P(k), P(k), 0, 16, P(out), None, st) == EINVAL          # q_len < 1
    assert call(ctx._h, P(q), P(k), P(k), 8, 7, P(out), None, st) == EINVAL           # kv_len < q_len
    assert call(ctx._h, NUL, P(k), P(k), 8, 16, P(out), None, st) == EINVAL           # null q
    assert call(ctx._h, P(q), P(k), NUL, 8, 16, P(out), None, st) == EINVAL           # null v
    assert call(ctx._h, P(q), P(k), P(k), 8, 16, NUL, None, st) == EINVAL             # null out
    assert call(ctx._h, P(q, 2), P(k), P(k), 7, 15, P(out), None, st) == EINVAL       # misaligned q
    assert call(ctx._h, P(q), P(k, 8), P(k), 7, 15, P(out), None, st) == EINVAL       # misaligned k
    assert call(ctx._h, P(q), P(k), P(k), 7, 15, P(out, 2), None, st) == EINVAL       # misaligned out
    assert call(ctx._h, P(q), P(k), P(k), 7, 15, P(out), P(f32, 4), st) == EINVAL     # misaligned out_f32
    with pytest.raises(N.MagicPigError):
        ctx.prefill_attend(q.float(), k, k)
    with pytest.raises(N.MagicPigError):
        ctx.prefill_attend(q[:, :16].contiguous(), k, k)
    with pytest.raises(N.MagicPigError):
        ctx.prefill_attend(q, k, k, out=torch.empty((8, 32, d), dtype=torch.float16, device=DEV))


def test_server_prefill_attention():
    """The FlashInfer-shaped entry point: output in q's dtype, the reference's keywords accepted, causal=False / HND refused."""
    from magicpig_b200.attnserver import LSHSparseAttnServer

    class Cfg:
        num_hidden_layers, num_key_value_heads, num_attention_heads, hidden_size = 2, 8, 32, 4096

    srv = LSHSparseAttnServer(Cfg(), K=K_, L=L_, max_length=1024, dense_layers=(0,), device=DEV)
    c = Case("mean", 300, 1000, 32, 8, seed=19)
    o64 = c.restate()
    got = srv.prefill_attention(q=c.q.half(), k=c.k.half(), v=c.v.half(), causal=True, allow_fp16_qk_reduction=True, kv_layout="NHD")
    assert got.dtype == torch.float16 and got.shape == (300, 32, d)
    ref = srv.ctx.prefill_attend(c.q.half().bfloat16(), c.k.half().bfloat16(), c.v.half().bfloat16())
    assert torch.equal(got, ref.half())
    assert (got.double() - o64).abs().max() <= 0.05 * o64.abs().max()   # fp16 inputs rounded to bf16: a loose sanity bound
    for kw in (dict(causal=False), dict(kv_layout="HND")):
        with pytest.raises(ValueError):
            srv.prefill_attention(c.q, c.k, c.v, **kw)


# ---- LlamaDecodeRunner.prefill ------------------------------------------------------------------------------------------------------
def _runner(B=1, t_max=0, seed=7):
    from magicpig_b200.llama_runner import LlamaDecodeRunner, LlamaShape
    shape = LlamaShape("tiny", 4, 512, 1024, 4, 2, 1000, 500000.0, 1e-5)   # d = 128, G = 2, layer 0 dense
    return LlamaDecodeRunner(shape, K_, L_, B, 4096, device=DEV, seed=seed, generation_buffer=256, dense_layers=(0,), fused=False,
                             max_chunk_tokens=t_max)


def _ref_forward(run, ids, dt):
    """A torch forward of the prompt ids (n,) with exact causal attention, in dtype dt: (last-token logits, [(k, v) per layer])."""
    sh, hs, Hq, Hkv, G = run.shape, run.shape.hidden_size, run.Hq_loc, run.Hkv_loc, run.Hq_loc // run.Hkv_loc
    n = ids.shape[0]
    cos, sin = run.cos[:n].to(dt)[:, None], run.sin[:n].to(dt)[:, None]

    def rope(x):
        return x * cos + torch.cat([-x[..., d // 2:], x[..., :d // 2]], -1) * sin

    h = run.embed[ids].to(dt)
    mask = torch.arange(n, device=DEV)[None, :] <= torch.arange(n, device=DEV)[:, None]
    kvs = []
    for lw in run.layers:
        W = {key: t.to(dt) for key, t in lw.items()}
        x = F.rms_norm(h, (hs,), W["ln1"], sh.rms_norm_eps)
        qkv = x @ W["wqkv"].T
        q = rope(qkv[:, :Hq * d].reshape(n, Hq, d))
        k = rope(qkv[:, Hq * d:(Hq + Hkv) * d].reshape(n, Hkv, d))
        v = qkv[:, (Hq + Hkv) * d:].reshape(n, Hkv, d)
        kvs.append((k, v))
        s = torch.einsum("nhd,khd->hnk", q, k.repeat_interleave(G, dim=1)) / math.sqrt(d)
        s = s.masked_fill(~mask[None], float("-inf"))
        p = torch.softmax(s.float() if dt == torch.bfloat16 else s, -1).to(dt)
        a = torch.einsum("hnk,khd->nhd", p, v.repeat_interleave(G, dim=1)).reshape(n, Hq * d)
        h = h + a @ W["wo"].T
        x = F.rms_norm(h, (hs,), W["ln2"], sh.rms_norm_eps)
        gu = x @ W["w_gate_up"].T
        it = run.it_loc
        h = h + (F.silu(gu[:, :it]) * gu[:, it:]) @ W["w_down"].T
    x = F.rms_norm(h[-1], (hs,), run.norm.to(dt), sh.rms_norm_eps)
    return (x @ run.lm_head.to(dt).T).double(), kvs


def _bar(r16, r64):
    return 2 * (r16.double() - r64).abs().max().item() + 1e-3


def _ids(n, seed):
    return torch.randint(0, 1000, (n,), generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)


def test_runner_prefill_vs_fp64():
    """P = 3 000 in chunks of 1 024 (a ragged last chunk): the last-token logits and every layer's K/V as handed to fill() are
    within 2x the bf16 torch forward's error + 1e-3 of an fp64 forward; pos and the server's lengths as synthetic_prefill leaves
    them."""
    P = 3000
    ids = _ids(P, 1)
    run = _runner()
    handed = []
    fill = run.server.fill
    run.server.fill = lambda layer, r, k, v, n: (handed.append((k.clone(), v.clone(), n)), fill(layer, r, k, v, n))[1]
    run.prefill(ids, chunk_size=1024)
    assert run.pos.tolist() == [P - 1]
    r64, kv64 = _ref_forward(run, ids, torch.float64)
    r16, kv16 = _ref_forward(run, ids, torch.bfloat16)
    err = (run.logits[0].double() - r64).abs().max().item()
    assert err <= _bar(r16, r64), f"logits: |runner - fp64| = {err:.3g} > {_bar(r16, r64):.3g}"
    assert len(handed) == 4
    for li, ((k, v, n), (k64, v64), (k16, v16)) in enumerate(zip(handed, kv64, kv16)):
        assert n == P and k.shape == (P, 2, d)
        for name, got, w64, w16 in (("k", k, k64, k16), ("v", v, v64, v16)):
            e = (got.double() - w64).abs().max().item()
            assert e <= _bar(w16, w64), f"layer {li} {name}: |runner - fp64| = {e:.3g} > {_bar(w16, w64):.3g}"
    assert run.server.ctx.error_flags() == 0


def test_runner_prefill_then_extend():
    """prefill(ids[:P]) + extend(ids[P:P+T]) and prefill(ids[:P+T]) both agree with the fp64 forward of ids[:P+T]."""
    P, T = 2000, 300
    ids = _ids(P + T, 2)
    r64, _ = _ref_forward(_runner(), ids, torch.float64)
    r16, _ = _ref_forward(_runner(), ids, torch.bfloat16)
    bar = _bar(r16, r64)
    a = _runner(t_max=256)
    a.prefill(ids[:P], chunk_size=1024)
    a.extend(ids[None, P:])
    assert a.pos.tolist() == [P + T - 1]
    b = _runner()
    b.prefill(ids, chunk_size=1024)
    for name, run in (("prefill + extend", a), ("prefill", b)):
        err = (run.logits[0].double() - r64).abs().max().item()
        assert err <= bar, f"{name}: |runner - fp64| = {err:.3g} > {bar:.3g}"
    assert a.server.ctx.error_flags() == 0


def test_runner_two_prompts_then_captured_step():
    """Two requests prefilled with different prompts, then a captured step(): no error flags, pos advanced from P_b - 1, and each
    request's prefill logits within the bar of its own fp64 forward."""
    lens = [1500, 2300]
    run = _runner(B=2)
    ids = [_ids(n, 3 + b) for b, n in enumerate(lens)]
    for b in range(2):
        run.prefill(ids[b], request=b, chunk_size=1024)
    assert run.pos.tolist() == [n - 1 for n in lens]
    for b in range(2):
        r64, _ = _ref_forward(run, ids[b], torch.float64)
        r16, _ = _ref_forward(run, ids[b], torch.bfloat16)
        err = (run.logits[b].double() - r64).abs().max().item()
        assert err <= _bar(r16, r64), f"request {b}: |runner - fp64| = {err:.3g}"
    run.ids.fill_(5)
    used = run.capture()
    run.replay()
    torch.cuda.synchronize()
    assert run.server.ctx.error_flags() == 0
    assert run.pos.tolist() == [n - 1 + used for n in lens]   # the warm-up steps and one replay
    assert bool(torch.isfinite(run.logits).all())


def test_runner_prefill_refusals():
    run = _runner()
    for n in (68, 4097):   # sink + local = 68; max_length = 4096
        with pytest.raises(ValueError):
            run.prefill(_ids(n, 4))
    assert run.pos.tolist() == [0]
