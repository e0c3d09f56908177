"""Chunk steps (mpig_plan_chunk / mpig_chunk_attend, `-m gpu`): T new prompt tokens per request attended exactly over the whole
context on the tensor cores, then folded into the store and the tables by spill_window().

  * fp32 outputs within 1e-3 (per row, relative to the row's max-norm) of an fp64 causal softmax over the stored rows, sparse
    and dense layers, tile-ragged T and store lengths, requests at different window lengths; dense with dense_tail_rows;
    T*G <= 32 agrees with mpig_dense_decode_tokens; the bf16 output is the fp32 output rounded half-up;
  * shared spill: each request sees its own spilled keys only;
  * chunk + spill leaves the state T single-token steps + spill leave: records, norms and table offsets bitwise, the items of every
    bucket as a set (the merge does not fix their order), and the next step's outputs bitwise;
  * shared spill: also equal to an exclusive-slot twin;
  * rewind after a chunk equals a chunk of the kept tokens (outputs and state); a captured chunk step replays to the eager outputs;
  * a sharp softmax, where P as plain bf16 would miss 1e-3;
  * refusals change nothing;
  * LlamaDecodeRunner.extend() of a ragged 300-token turn against a torch forward of the same model in fp64.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from magicpig_b200 import _native as N
from magicpig_b200 import synth
from tests.support.fp64 import assert_rounded_half_up, causal_ref, centred, rel_rows
from tests.support.library import DEV, NL, NS, assert_tables_equal, d, lsh_tables, two_layer_context

pytestmark = pytest.mark.gpu
K_, L_ = 6, 16


class Setup:
    """Layer 0 dense, layer 1 sparse.  Slot c's store holds n keys; request b's window w[b] rows and its dense cache p[b] rows."""

    def __init__(self, B, n=1337, w=None, p=None, C=0, shared_spill=False, tail=0, gen=320, M=4096, t_max=512, Hq=32, Hkv=8, seed=0,
                 one_prompt=False):
        """one_prompt: every slot is filled with the same prompt (drawn as for one slot), so that C = B gives the exclusive-slot twin
        of a context with C = 1."""
        self.B, self.Hq, self.Hkv, self.G = B, Hq, Hkv, Hq // Hkv
        self.ctx = ctx = two_layer_context(K_, L_, Hq, Hkv, B, M, gen, synth.make_hash_func(d, K_, L_, seed=seed), dict(out_f32=1),
                                           alloc_dense_kv=True, num_contexts=C, dense_tail_rows=tail, shared_spill=shared_spill)
        ctx.reserve_chunk_tokens(t_max)
        self.g = g = torch.Generator(device=DEV).manual_seed(seed + 1)
        rnd = lambda *s: torch.randn(s, generator=g, device=DEV).bfloat16()   # noqa: E731
        nslots = C or B
        self.w = w or [NS + NL] * B
        self.p = p or [900] * B
        ndraw = 1 if one_prompt else nslots
        self.sk, self.sv = rnd(ndraw, Hkv, n, d), rnd(ndraw, Hkv, n, d)
        if one_prompt:
            self.sk, self.sv = self.sk.expand(nslots, -1, -1, -1), self.sv.expand(nslots, -1, -1, -1)
        self.n = n
        for c in range(nslots):   # request c is bound to slot c at creation
            ctx.attn_fill(1, c, self.sk[c].contiguous(), self.sv[c].contiguous(), self.sk[c].float().norm(dim=-1).contiguous())
            ctx.lsh_build(1, c, ctx.hash_keys(self.sk[c].contiguous()))
            if one_prompt and c > 0:
                self.dk[c], self.dv[c] = self.dk[0], self.dv[0]
            else:
                self._dense(c, rnd)
            ctx.dense_fill(0, c, self.dk[c].contiguous(), self.dv[c].contiguous(), self.p[c])
        for b in range(nslots, B):
            ctx.fork(b % nslots, b)
        self.avg = rnd(B, Hkv, d) * 0.1
        self.wk, self.wv = [], []
        for b in range(B):
            self.wk.append(rnd(Hkv, self.w[b], d))
            self.wv.append(rnd(Hkv, self.w[b], d))
            ctx.window_fill(1, b, self.avg[b].contiguous(), self.wk[b], self.wv[b])
        torch.cuda.synchronize()

    def _dense(self, c, rnd):
        self.dk = getattr(self, "dk", {})
        self.dv = getattr(self, "dv", {})
        self.dk[c], self.dv[c] = rnd(self.p[c], self.Hkv, d), rnd(self.p[c], self.Hkv, d)
        return self.dk[c], self.dv[c]

    def qkv(self, T):
        g = self.g
        return (torch.randn((self.B, T, self.Hq, d), generator=g, device=DEV).bfloat16(),
                torch.randn((self.B, T, self.Hkv, d), generator=g, device=DEV).bfloat16(),
                torch.randn((self.B, T, self.Hkv, d), generator=g, device=DEV).bfloat16())

    def chunk(self, layer, T, q, k, v):
        out = self.ctx.chunk_attend(layer, T, q, k, v)
        return out, self.ctx.last_out_f32().reshape(self.B, T, self.Hq, d)


def check(f32, ref, what):
    """Per row (token, q-head): max|out_f32 - fp64| <= 1e-3 max|fp64|."""
    err = rel_rows(f32, ref)
    assert err <= 1e-3, f"{what}: max|out_f32 - fp64| / max|fp64| = {err:.3g}"


def sparse_ref(s, b, h, q, k, v, store_keys=None):
    """fp64 output of request b, kv-head h, for a chunk on the sparse layer: store rows (all of the slot unless given), window rows,
    the chunk's centred rows."""
    G = s.G
    sk, sv = store_keys if store_keys is not None else (s.sk[b % (s.ctx.C)][h], s.sv[b % (s.ctx.C)][h])
    kctx = torch.cat([sk, s.wk[b][h]], 0)
    vctx = torch.cat([sv, s.wv[b][h]], 0)
    return causal_ref(q[b, :, h * G:(h + 1) * G], kctx, vctx, centred(k[b, :, h], s.avg[b, h]), v[b, :, h])


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("T", [1, 7, 64, 257])
def test_chunk_sparse_and_dense_vs_fp64(cuda_lib, B, T):
    s = Setup(B, n=1337, w=[NS + NL + 13 * b for b in range(B)], p=[900 + 37 * b for b in range(B)], seed=B * 1000 + T)
    s.ctx.plan_chunk(T)
    q, k, v = s.qkv(T)
    out1, f1 = s.chunk(1, T, q, k, v)
    q0, k0, v0 = s.qkv(T)
    out0, f0 = s.chunk(0, T, q0, k0, v0)
    for out, f, layer in ((out1, f1, "sparse"), (out0, f0, "dense")):
        assert_rounded_half_up(out, f, f"{layer} chunk")
    for b in range(B):
        for h in range(s.Hkv):
            check(f1[b, :, h * s.G:(h + 1) * s.G], sparse_ref(s, b, h, q, k, v), f"sparse b={b} h={h}")
            ref0 = causal_ref(q0[b, :, h * s.G:(h + 1) * s.G], s.dk[b][:, h], s.dv[b][:, h], k0[b, :, h], v0[b, :, h])
            check(f0[b, :, h * s.G:(h + 1) * s.G], ref0, f"dense b={b} h={h}")
    assert s.ctx.error_flags() == 0


def test_chunk_dense_tail_rows_and_tokens_agree(cuda_lib):
    """Shared dense prefix (dense_tail_rows): three requests on one slot; and for T*G <= 32 the chunk step agrees with the
    verification step's dense kernel."""
    s = Setup(3, C=1, tail=600, p=[1111], seed=5)
    s.ctx.reserve_query_tokens(8)
    for T in (8, 100):
        s.ctx.plan_chunk(T)
        q, k, v = s.qkv(T)
        _, f0 = s.chunk(0, T, q, k, v)
        for b in range(3):
            for h in range(s.Hkv):
                ref = causal_ref(q[b, :, h * s.G:(h + 1) * s.G], s.dk[0][:, h], s.dv[0][:, h], k[b, :, h], v[b, :, h])
                check(f0[b, :, h * s.G:(h + 1) * s.G], ref, f"tail T={T} b={b} h={h}")
        s.ctx.rewind(torch.full((3,), T, dtype=torch.int32, device=DEV))
        if T * s.G <= 32:
            s.ctx.plan(T)
            s.ctx.dense_decode_tokens(0, T, q, k, v)
            ft = s.ctx.last_out_f32().reshape(f0.shape)
            assert (ft - f0).abs().max().item() <= 1e-5
            s.ctx.rewind(torch.full((3,), T, dtype=torch.int32, device=DEV))


def _generate(s, steps, seed):
    """`steps` single-token steps on the sparse layer with per-request rows; returns the centred rows per request (Hkv, steps, d)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    rows = []
    for _ in range(steps):
        q = torch.randn((s.B, s.Hq, 1, d), generator=g, device=DEV).bfloat16()
        k = torch.randn((s.B, s.Hkv, 1, d), generator=g, device=DEV).bfloat16()
        v = torch.randn((s.B, s.Hkv, 1, d), generator=g, device=DEV).bfloat16()
        s.ctx.plan()
        s.ctx.decode(1, q, k, v)
        rows.append((k[:, :, 0], v[:, :, 0]))
    kk = torch.stack([r[0] for r in rows], 2)   # (B, Hkv, steps, d)
    vv = torch.stack([r[1] for r in rows], 2)
    return [centred(kk[b], s.avg[b][:, None]) for b in range(s.B)], [vv[b] for b in range(s.B)]


def test_chunk_shared_spill_sees_own_keys(cuda_lib):
    """Three requests on one slot, each spilling 40 different keys: each chunk output equals that of an exclusive-slot twin holding
    the prompt and the request's own spilled keys (fp32 up to summation order) and fp64."""
    s = Setup(3, C=1, shared_spill=True, seed=11, one_prompt=True)
    twin = Setup(3, seed=11, one_prompt=True)
    gk, gv = _generate(s, 40, seed=12)
    _generate(twin, 40, seed=12)
    spilled = s.ctx.spill_window().tolist()
    assert spilled == [40, 40, 40] and twin.ctx.spill_window().tolist() == spilled
    # windows after the spill: the sink rows, then the newest NL of (local + generated)
    for b in range(3):
        allk = torch.cat([s.wk[b], gk[b]], 1)
        allv = torch.cat([s.wv[b], gv[b]], 1)
        s.wk[b] = torch.cat([allk[:, :NS], allk[:, -NL:]], 1)
        s.wv[b] = torch.cat([allv[:, :NS], allv[:, -NL:]], 1)
        s.__dict__.setdefault("priv", []).append((allk[:, NS:-NL], allv[:, NS:-NL]))
    T = 64
    s.ctx.plan_chunk(T)
    q, k, v = s.qkv(T)
    _, f1 = s.chunk(1, T, q, k, v)
    twin.ctx.plan_chunk(T)
    _, ft = twin.chunk(1, T, q, k, v)
    assert (f1 - ft).abs().max().item() <= 1e-5, "shared spill != exclusive-slot twin"
    ks, vs, _ = s.ctx.read_cache(1)
    kt, _, _ = twin.ctx.read_cache(1)
    for b in range(3):
        lo = s.n + 40 * b
        assert torch.equal(ks[0, :, lo:lo + 40], s.priv[b][0])
        assert torch.equal(kt[b, :, s.n:s.n + 40], s.priv[b][0])
        for h in range(s.Hkv):
            store = (torch.cat([s.sk[0][h], s.priv[b][0][h]], 0), torch.cat([s.sv[0][h], s.priv[b][1][h]], 0))
            check(f1[b, :, h * s.G:(h + 1) * s.G], sparse_ref(s, b, h, q, k, v, store), f"shared spill b={b} h={h}")


@pytest.mark.parametrize("shared", [False, True])
def test_chunk_then_spill_equals_single_token_steps(cuda_lib, shared):
    kw = dict(C=1, shared_spill=True) if shared else {}
    B, T = (3 if shared else 2), 40
    a, b_ = Setup(B, seed=21, **kw), Setup(B, seed=21, **kw)
    q, k, v = a.qkv(T)
    a.ctx.plan_chunk(T)
    a.ctx.chunk_attend(1, T, q, k, v)
    a.ctx.chunk_attend(0, T, q, k, v)
    for t in range(T):
        b_.ctx.plan()
        b_.ctx.decode(1, q[:, t].contiguous(), k[:, t].contiguous(), v[:, t].contiguous())
        b_.ctx.dense_decode(0, q[:, t].contiguous(), k[:, t].contiguous(), v[:, t].contiguous())
    assert a.ctx.spill_window().tolist() == b_.ctx.spill_window().tolist() == [T] * B
    for x, y in zip(a.ctx.read_cache(1), b_.ctx.read_cache(1)):
        assert torch.equal(x, y)
    assert_tables_equal(lsh_tables(a.ctx, 1), lsh_tables(b_.ctx, 1))
    # the windows, dense rows and lengths: the next step's outputs are bitwise equal
    qx, kx, vx = a.qkv(1)
    for s in (a, b_):
        s.ctx.plan()
    for layer, fn in ((1, "decode"), (0, "dense_decode")):
        oa = getattr(a.ctx, fn)(layer, qx[:, 0].contiguous(), kx[:, 0].contiguous(), vx[:, 0].contiguous()).clone()
        ob = getattr(b_.ctx, fn)(layer, qx[:, 0].contiguous(), kx[:, 0].contiguous(), vx[:, 0].contiguous()).clone()
        assert torch.equal(oa, ob), fn
    assert a.ctx.error_flags() == 0 and b_.ctx.error_flags() == 0


def test_chunk_rewind_equals_chunk_of_kept_tokens(cuda_lib):
    """rewind(T - n_b) after a chunk of T: request b's kept outputs and its state equal those of a chunk of n_b tokens (for n_b = 0:
    no chunk at all).  The state is compared through the next single-token step's outputs on both layers, bitwise."""
    T, kept = 50, [50, 30, 0]
    s = Setup(3, seed=33)
    q, k, v = s.qkv(T)
    qx, kx, vx = (t[:, 0].contiguous() for t in s.qkv(1))
    s.ctx.plan_chunk(T)
    _, f1 = s.chunk(1, T, q, k, v)
    f1 = f1.clone()
    _, f0 = s.chunk(0, T, q, k, v)
    s.ctx.rewind(torch.tensor([T - n for n in kept], dtype=torch.int32, device=DEV))
    s.ctx.plan()
    nxt = (s.ctx.decode(1, qx, kx, vx).clone(), s.ctx.dense_decode(0, qx, kx, vx).clone())
    for b, n in enumerate(kept):
        twin = Setup(3, seed=33)
        if n > 0:
            twin.ctx.plan_chunk(n)
            _, t1 = twin.chunk(1, n, q[:, :n].contiguous(), k[:, :n].contiguous(), v[:, :n].contiguous())
            t1 = t1.clone()
            _, t0 = twin.chunk(0, n, q[:, :n].contiguous(), k[:, :n].contiguous(), v[:, :n].contiguous())
            assert (f1[b, :n] - t1[b]).abs().max().item() <= 1e-5 and (f0[b, :n] - t0[b]).abs().max().item() <= 1e-5, f"b={b}"
        twin.ctx.plan()
        tn = (twin.ctx.decode(1, qx, kx, vx), twin.ctx.dense_decode(0, qx, kx, vx))
        assert torch.equal(nxt[0][b], tn[0][b]) and torch.equal(nxt[1][b], tn[1][b]), f"state of request {b} after the rewind"


def test_chunk_rewind_then_next_chunk(cuda_lib):
    s = Setup(3, seed=31)
    T1, T2, drop = 50, 30, [0, 20, 50]
    q, k, v = s.qkv(T1)
    s.ctx.plan_chunk(T1)
    s.ctx.chunk_attend(1, T1, q, k, v)
    s.ctx.chunk_attend(0, T1, q, k, v)
    s.ctx.rewind(torch.tensor(drop, dtype=torch.int32, device=DEV))
    for b in range(3):   # the kept rows join the context of the next chunk
        kept = T1 - drop[b]
        s.wk[b] = torch.cat([s.wk[b], centred(k[b, :kept].transpose(0, 1), s.avg[b][:, None])], 1)
        s.wv[b] = torch.cat([s.wv[b], v[b, :kept].transpose(0, 1)], 1)
        s.dk[b] = torch.cat([s.dk[b], k[b, :kept]], 0)
        s.dv[b] = torch.cat([s.dv[b], v[b, :kept]], 0)
    q2, k2, v2 = s.qkv(T2)
    s.ctx.plan_chunk(T2)
    _, f1 = s.chunk(1, T2, q2, k2, v2)
    _, f0 = s.chunk(0, T2, q2, k2, v2)
    for b in range(3):
        for h in range(s.Hkv):
            check(f1[b, :, h * s.G:(h + 1) * s.G], sparse_ref(s, b, h, q2, k2, v2), f"sparse b={b}")
            ref0 = causal_ref(q2[b, :, h * s.G:(h + 1) * s.G], s.dk[b][:, h], s.dv[b][:, h], k2[b, :, h], v2[b, :, h])
            check(f0[b, :, h * s.G:(h + 1) * s.G], ref0, f"dense b={b}")


def test_chunk_captured_replays_to_eager_and_refusals(cuda_lib):
    s = Setup(2, seed=41)
    ctx, T = s.ctx, 96
    q, k, v = s.qkv(T)
    o1, o0 = torch.empty((2, T, s.Hq * d), dtype=torch.bfloat16, device=DEV), torch.empty((2, T, s.Hq * d), dtype=torch.bfloat16, device=DEV)
    drop_all = torch.full((2,), T, dtype=torch.int32, device=DEV)
    ctx.plan_chunk(T)
    ctx.chunk_attend(1, T, q, k, v, o1)
    ctx.chunk_attend(0, T, q, k, v, o0)
    e1, e0, ef = o1.clone(), o0.clone(), ctx.last_out_f32()
    ctx.rewind(drop_all)
    # refusals (nothing changes: the eager chunk below still sees the same state)
    with pytest.raises(N.MagicPigError):
        ctx.plan_chunk(513)                       # above the reserve
    with pytest.raises(N.MagicPigError):
        ctx.plan_chunk(ctx.Wcap - (NS + NL) + 1)  # the window cannot hold it
    ctx.reserve_query_tokens(2)
    ctx.plan(2)
    with pytest.raises(N.MagicPigError):
        ctx.chunk_attend(1, 2, *s.qkv(2))        # a verification step is pending
    ctx.rewind(torch.full((2,), 2, dtype=torch.int32, device=DEV))
    ctx.plan_chunk(2)
    with pytest.raises(N.MagicPigError):
        ctx.decode_tokens(1, 2, *s.qkv(2))       # a chunk step is pending
    with pytest.raises(N.MagicPigError):
        ctx.dense_decode_tokens(0, 2, *s.qkv(2))
    ctx.rewind(torch.full((2,), 2, dtype=torch.int32, device=DEV))
    # capture
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        ctx.plan_chunk(T)
        ctx.chunk_attend(1, T, q, k, v, o1)
        ctx.chunk_attend(0, T, q, k, v, o0)
    o1.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert (ctx.last_out_f32() - ef).abs().max().item() <= 1e-5
    assert (o1.float() - e1.float()).abs().max().item() <= 2 ** -6 and (o0.float() - e0.float()).abs().max().item() <= 2 ** -6
    with pytest.raises(N.MagicPigError):
        ctx.reserve_chunk_tokens(1024)            # the scratch would move under the graph
    assert ctx.get_info("chunk_tokens_max") == 512
    assert ctx.error_flags() == 0


def test_chunk_refuses_dense_capacity(cuda_lib):
    """dense_tail_rows = 50: a chunk of 51 does not fit the tails (the windows would hold it): refused, nothing changed."""
    s = Setup(3, C=1, tail=50, p=[700], seed=51)
    with pytest.raises(N.MagicPigError, match="dense KV cache is full"):
        s.ctx.plan_chunk(51)
    T = 50
    s.ctx.plan_chunk(T)
    q, k, v = s.qkv(T)
    _, f0 = s.chunk(0, T, q, k, v)
    for b in range(3):
        for h in range(s.Hkv):
            ref = causal_ref(q[b, :, h * s.G:(h + 1) * s.G], s.dk[0][:, h], s.dv[0][:, h], k[b, :, h], v[b, :, h])
            check(f0[b, :, h * s.G:(h + 1) * s.G], ref, f"b={b} h={h}")
    assert s.ctx.error_flags() == 0


def test_chunk_sharp_softmax_vs_fp64(cuda_lib):
    """Queries 4x the usual scale (a few keys take most of the probability), where P rounded to plain bf16 misses 1e-3 (see
    tests/test_chunk_cpu.py): the hi + lo split keeps the bar."""
    s = Setup(1, n=8000, M=9000, seed=61)
    T = 64
    s.ctx.plan_chunk(T)
    q, k, v = s.qkv(T)
    q = (q.float() * 4).bfloat16()
    _, f1 = s.chunk(1, T, q, k, v)
    _, f0 = s.chunk(0, T, q, k, v)
    for h in range(s.Hkv):
        check(f1[0, :, h * s.G:(h + 1) * s.G], sparse_ref(s, 0, h, q, k, v), f"sparse h={h}")
        ref0 = causal_ref(q[0, :, h * s.G:(h + 1) * s.G], s.dk[0][:, h], s.dv[0][:, h], k[0, :, h], v[0, :, h])
        check(f0[0, :, h * s.G:(h + 1) * s.G], ref0, f"dense h={h}")


def test_chunk_needs_reserve(cuda_lib):
    from magicpig_b200.ops import Context
    ctx = Context(K_, L_, 2, 32, 8, d, 1, 1024, NS, NL, 64, dense_layers=[0], alloc_dense_kv=True, device=DEV)
    assert ctx.get_info("chunk_tokens_max") == 0
    with pytest.raises(N.MagicPigError):
        ctx.plan_chunk(1)


# ---- LlamaDecodeRunner.extend ------------------------------------------------------------------------------------------------
def _runner(gen, t_max, P, seed=7):
    from magicpig_b200.llama_runner import LlamaDecodeRunner, LlamaShape
    shape = LlamaShape("tiny", 4, 512, 1024, 4, 2, 1000, 500000.0, 1e-5)
    run = LlamaDecodeRunner(shape, K_, L_, 2, 2048, device=DEV, seed=seed, generation_buffer=gen, dense_layers=(0,),
                            fused=False, max_chunk_tokens=t_max)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    pref = []
    for layer in range(4):
        kv = []
        for b in range(2):
            k = torch.randn((P, 2, d), generator=g, device=DEV).bfloat16()
            v = torch.randn((P, 2, d), generator=g, device=DEV).bfloat16()
            run.server.alloc_buffer(P)
            run.server.fill(layer, b, k, v, P)
            run.server.build_table(layer, b, P)
            kv.append((k, v))
        pref.append(kv)
    run.pos.fill_(P - 1)
    torch.cuda.synchronize()
    return run, pref


def _ref_logits(run, ids, pref, b, P, dt):
    """A torch forward of the turn ids (n,) of request b with exact causal attention over its prefill K/V, in dtype dt."""
    sh, hs, Hq, Hkv, G = run.shape, run.shape.hidden_size, run.Hq_loc, run.Hkv_loc, run.Hq_loc // run.Hkv_loc
    n = ids.shape[0]
    pos = P + torch.arange(n, device=DEV)
    cos, sin = run.cos[pos].to(dt)[:, None], run.sin[pos].to(dt)[:, None]

    def rope(x):
        return x * cos + torch.cat([-x[..., d // 2:], x[..., :d // 2]], -1) * sin

    h = run.embed[ids].to(dt)
    mask = torch.arange(P + n, device=DEV)[None, :] <= (P + torch.arange(n, device=DEV))[:, None]
    for li, lw in enumerate(run.layers):
        W = {key: t.to(dt) for key, t in lw.items()}
        x = F.rms_norm(h, (hs,), W["ln1"], sh.rms_norm_eps)
        qkv = x @ W["wqkv"].T
        q = rope(qkv[:, :Hq * d].reshape(n, Hq, d))
        k = rope(qkv[:, Hq * d:(Hq + Hkv) * d].reshape(n, Hkv, d))
        v = qkv[:, (Hq + Hkv) * d:].reshape(n, Hkv, d)
        Kx = torch.cat([pref[li][b][0].to(dt), k], 0).repeat_interleave(G, dim=1)
        Vx = torch.cat([pref[li][b][1].to(dt), v], 0).repeat_interleave(G, dim=1)
        s = torch.einsum("nhd,khd->hnk", q, Kx) / math.sqrt(d)
        p = torch.softmax(s.masked_fill(~mask[None], float("-inf")).float() if dt == torch.bfloat16 else
                          s.masked_fill(~mask[None], float("-inf")), -1).to(dt)
        a = torch.einsum("hnk,khd->nhd", p, Vx).reshape(n, Hq * d)
        h = h + a @ W["wo"].T
        x = F.rms_norm(h, (hs,), W["ln2"], sh.rms_norm_eps)
        gu = x @ W["w_gate_up"].T
        it = run.it_loc
        h = h + (F.silu(gu[:, :it]) * gu[:, it:]) @ W["w_down"].T
    x = F.rms_norm(h[-1], (hs,), run.norm.to(dt), sh.rms_norm_eps)
    return (x @ run.lm_head.to(dt).T).double()


def test_runner_extend_ragged_turn(cuda_lib):
    P, lengths = 500, [300, 217]
    ids = torch.randint(0, 1000, (2, 300), generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)
    results = []
    for gen, t_max in ((128, 256), (512, 512)):   # several chunks with spills inside the turn; one chunk
        run, pref = _runner(gen, t_max, P)
        run.extend(ids, torch.tensor(lengths))
        assert run.pos.tolist() == [P - 1 + n for n in lengths]
        results.append(run.logits.double().clone())
        if gen == 128:
            run.ids.fill_(5)
            run.step()
            assert run.server.ctx.error_flags() == 0
            many_run, many_pref = run, pref
    for b, n in enumerate(lengths):
        r64 = _ref_logits(many_run, ids[b, :n], many_pref, b, P, torch.float64)
        r16 = _ref_logits(many_run, ids[b, :n], many_pref, b, P, torch.bfloat16)
        bar = 2 * (r16 - r64).abs().max().item() + 1e-3
        for name, got in zip(("several chunks", "one chunk"), results):
            err = (got[b] - r64).abs().max().item()
            assert err <= bar, f"{name} b={b}: |runner - fp64| = {err:.3g} > {bar:.3g}"
