"""Sampling on the device (mpig_aux_sample, csrc/aux_sample.cu) against the restatement of its contract in
tests/support/sample_rule.py, and LlamaDecodeRunner.generate() end to end.

Exactness: for every row, (1) the kernel's fp32 weights are within the derived bound of fp64 exp((l - m) / T); (2) the restatement's
integer stages on the kernel's own weights give the kernel's token and debug output bitwise; (3) the restatement on fp64 weights
gives the same token, except a draw whose nucleus boundary or target lies within the bound of a boundary, which may take only
the tokens sample_rule.allowed_tokens admits."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

from magicpig_b200.ops import sample
from tests.support import sample_rule as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TEMPS = (0.0, 0.1, 0.6, 1.0, 2.0)
TOPS = (0.0, 0.5, 0.9, 1.0)
MPIG_EINVAL = -1   # include/magicpig_b200.h


def _logits(regime, B, V, seed):
    g = torch.Generator().manual_seed(seed)
    if regime == "flat":      # the nucleus is most of the vocabulary
        l = torch.randn((B, V), generator=g) * 0.05
    elif regime == "peaked":  # 1-3 tokens hold almost all the mass
        l = torch.randn((B, V), generator=g)
        for b in range(B):
            k = 1 + b % 3
            l[b, torch.randint(0, V, (k,), generator=g)] = 25.0 + torch.rand(k, generator=g)
    elif regime == "ties":    # integer logits: many exact ties, thresholds inside tie groups
        l = torch.round(torch.randn((B, V), generator=g) * 1.5)
    elif regime == "masked":  # most of the vocabulary at -inf
        l = torch.randn((B, V), generator=g) * 2
        l[torch.rand((B, V), generator=g) < 0.9] = float("-inf")
    return l.float()


def _params(B, shift):
    T = torch.tensor([TEMPS[(b + shift) % len(TEMPS)] for b in range(B)], dtype=torch.float32)
    p = torch.tensor([TOPS[(b // len(TEMPS) + b + shift) % len(TOPS)] for b in range(B)], dtype=torch.float32)
    return T, p


def _run(l, T, p, seed, off, dbg=True):
    B, V = l.shape
    offset = torch.tensor([off], dtype=torch.int64, device=DEV)
    debug = torch.zeros((B, 5), dtype=torch.int64, device=DEV) if dbg else None
    debug_w = torch.full((B, V), -1.0, device=DEV) if dbg else None
    status = torch.zeros(((B + 31) // 32,), dtype=torch.int32, device=DEV)
    ids = sample(l.to(DEV), T.to(DEV), p.to(DEV), seed, offset, status=status, debug=debug, debug_w=debug_w)
    torch.cuda.synchronize()
    assert int(offset.item()) == off, "the kernel wrote the offset"
    return ids.cpu(), (debug.cpu() if dbg else None), (debug_w.cpu() if dbg else None), status.cpu()


@pytest.mark.parametrize("V", [128256, 32000])
@pytest.mark.parametrize("B", [1, 8, 32])
@pytest.mark.parametrize("regime", ["flat", "peaked", "ties", "masked"])
def test_exact_against_restatement(cuda_lib, V, B, regime):
    seed, off = 1234 + B, 7 + V % 13
    l = _logits(regime, B, V, seed=V + B)
    T, p = _params(B, shift={"flat": 0, "peaked": 1, "ties": 2, "masked": 3}[regime])
    ids, dbg, dbg_w, status = _run(l, T, p, seed, off)
    assert int(status.sum()) == 0
    for b in range(B):
        row, t, pp = l[b].numpy(), float(T[b]), float(p[b])
        want, want_dbg = R.sample_row(row, t, pp, seed, off, b)
        if R.row_kind(row, t) is not None:   # greedy: the first argmax
            assert int(ids[b]) == want and tuple(dbg[b].tolist()) == want_dbg, (b, t)
            continue
        w64 = R.weights_fp64(row, t)
        wk = dbg_w[b].double().numpy()
        rel = R.weight_rel_bound(row, t)
        # plus 2^-60 absolute for fp32's subnormal range, far below the 2^-40 quantum of W
        assert np.all(np.abs(wk - w64) <= w64 * rel + 2.0 ** -60), f"row {b}: fp32 weights outside the bound, T={t}"
        tok_k, dbg_k = R.sample_row(row, t, pp, seed, off, b, W=R.fixed_point(wk))
        assert int(ids[b]) == tok_k, f"row {b}: kernel {int(ids[b])} vs restatement on its weights {tok_k} (T={t}, p={pp})"
        assert tuple(dbg[b].tolist()) == dbg_k, f"row {b}: debug {dbg[b].tolist()} vs {dbg_k}"
        if int(ids[b]) != want:
            allowed = R.allowed_tokens(row, t, pp, R.draw_word(seed, off, b), R.fixed_point(w64), rel)
            assert int(ids[b]) in allowed and want in allowed, f"row {b}: {int(ids[b])} vs fp64 {want} outside the bound"


def test_per_request_parameters_in_one_batch(cuda_lib):
    """Every (T, p) pair of the grid in one batch of 20 rows over the same logits: each row follows its own parameters."""
    V = 50257
    pairs = [(t, q) for t in TEMPS for q in TOPS]
    l = torch.randn((1, V), generator=torch.Generator().manual_seed(5)).float().repeat(len(pairs), 1) * 3
    T = torch.tensor([t for t, _ in pairs])
    p = torch.tensor([q for _, q in pairs])
    ids, dbg, dbg_w, _ = _run(l, T, p, 99, 3)
    for b, (t, q) in enumerate(pairs):
        row = l[b].numpy()
        W = R.fixed_point(dbg_w[b].double().numpy()) if t > 0 else None
        assert (int(ids[b]), tuple(dbg[b].tolist())) == R.sample_row(row, t, q, 99, 3, b, W=W), (t, q)


def test_chi_square_against_nucleus(cuda_lib):
    """200 000 draws (1 000 rows x 200 offsets) of one small-support row pass a chi-square test against the exact nucleus
    probabilities W_i / S_keep; the same test rejects the un-truncated distribution W_i / S."""
    V, rows, offs = 64, 1000, 200
    base = torch.full((V,), float("-inf"))
    base[:12] = torch.tensor([2.0, 1.7, 1.5, 1.2, 1.0, 0.8, 0.5, 0.3, 0.0, -0.4, -0.9, -1.5])
    l = base.repeat(rows, 1)
    T = torch.full((rows,), 0.8)
    p = torch.full((rows,), 0.75)
    counts = np.zeros(V, dtype=np.int64)
    ids0, _, dbg_w, _ = _run(l, T, p, 2024, 0)
    W = R.fixed_point(dbg_w[0].double().numpy())
    keep = R.sample_from_weights(W, 0.75, 0)[2]
    for off in range(offs):
        ids = ids0 if off == 0 else _run(l, T, p, 2024, off, dbg=False)[0]
        counts += np.bincount(ids.numpy(), minlength=V)
    assert counts.sum() == rows * offs
    assert counts[~keep].sum() == 0, "a token outside the nucleus was drawn"
    k = np.nonzero(keep)[0]
    exp_nucleus = W[k] / W[k].sum() * counts.sum()
    p_ok = stats.chisquare(counts[k], exp_nucleus).pvalue
    assert p_ok > 1e-4, f"chi-square against the nucleus: p = {p_ok:.3g}"
    pos = W > 0
    exp_full = W[pos] / W[pos].sum() * counts.sum()
    p_full = stats.chisquare(counts[pos], exp_full).pvalue
    assert p_full < 1e-4, f"the un-truncated distribution was not rejected: p = {p_full:.3g}"


def test_deterministic_and_offset_sensitive(cuda_lib):
    l = _logits("flat", 8, 32000, 1)
    T, p = torch.full((8,), 1.0), torch.full((8,), 0.95)
    a = _run(l, T, p, 5, 11)[0]
    b = _run(l, T, p, 5, 11)[0]
    c = _run(l, T, p, 5, 12)[0]
    d = _run(l, T, p, 6, 11)[0]
    assert torch.equal(a, b)
    assert not torch.equal(a, c) and not torch.equal(a, d)


def test_capture_replays_equal_eager_offsets(cuda_lib):
    """A captured sample + offset.add_(1): replay k equals an eager call at offset k, with parameters changed between replays."""
    B, V = 8, 128256
    l = _logits("flat", B, V, 3).to(DEV)
    T = torch.full((B,), 1.0, device=DEV)
    p = torch.full((B,), 0.9, device=DEV)
    off = torch.zeros(1, dtype=torch.int64, device=DEV)
    ids = torch.zeros((B, 1), dtype=torch.int64, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sample(l, T, p, 77, off, ids_out=ids)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        sample(l, T, p, 77, off, ids_out=ids)
        off.add_(1)
    off.zero_()
    for k in range(4):
        if k == 2:
            T.fill_(0.5)
            p.fill_(0.5)
        g.replay()
        torch.cuda.synchronize()
        eager = sample(l, T, p, 77, torch.tensor([k], dtype=torch.int64, device=DEV))
        assert torch.equal(ids[:, 0], eager), k
    assert int(off.item()) == 4


def test_status_bits_and_token_zero(cuda_lib):
    B, V = 40, 1000
    l = torch.randn((B, V))
    l[3, 17] = float("nan")
    l[5] = float("-inf")
    l[33, 2] = float("inf")
    T = torch.tensor([1.0 if b % 2 else 0.0 for b in range(B)])
    p = torch.full((B,), 0.9)
    ids, dbg, _, status = _run(l, T, p, 1, 0)
    assert status.tolist() == [(1 << 3) | (1 << 5), 1 << 1]
    for b in (3, 5, 33):
        assert int(ids[b]) == 0 and dbg[b].tolist() == [0] * 5


def test_bookkeeping(cuda_lib):
    """ids_out stride, the record, EOS and max_new."""
    B, V = 3, 500
    l = torch.full((B, V), -5.0)
    l[0, 7] = l[1, 9] = l[2, 11] = 10.0
    l = l.to(DEV)
    T, p = torch.zeros(B, device=DEV), torch.ones(B, device=DEV)
    ids = torch.zeros((B, 4), dtype=torch.int64, device=DEV)
    tok = torch.zeros((B, 2), dtype=torch.int32, device=DEV)
    cnt = torch.zeros(B, dtype=torch.int32, device=DEV)
    done = torch.zeros(B, dtype=torch.int32, device=DEV)
    done[2] = 1
    off = torch.zeros(1, dtype=torch.int64, device=DEV)
    sample(l, T, p, 0, off, ids_out=ids, tokens_out=tok, count=cnt, done=done, eos_token_ids=[9])
    assert ids[:, 0].tolist() == [7, 9, 11] and ids[:, 1:].abs().sum() == 0
    assert tok.tolist() == [[7, 0], [9, 0], [0, 0]] and cnt.tolist() == [1, 1, 0] and done.tolist() == [0, 1, 1]
    sample(l, T, p, 0, off, ids_out=ids, tokens_out=tok, count=cnt, done=done, eos_token_ids=[9])
    assert tok.tolist() == [[7, 7], [9, 0], [0, 0]] and cnt.tolist() == [2, 1, 0] and done.tolist() == [1, 1, 1]


def test_refusals(cuda_lib):
    lib = cuda_lib
    l = torch.zeros((2, 409601), device=DEV)
    T = torch.ones(2, device=DEV)
    off = torch.zeros(1, dtype=torch.int64, device=DEV)
    tok = torch.zeros((2, 4), dtype=torch.int32, device=DEV)
    P = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    eos = (ctypes.c_int32 * 9)(*range(9))

    def call(logits=P(l), B=2, V=1000, ld=409601, temp=P(T), top=P(T), offset=P(off), ids=None, stride=1, tokens=None, count=None,
             done=None, max_new=0, n_eos=0):
        return lib.mpig_aux_sample(logits, B, V, ld, temp, top, 0, offset, ids, stride, tokens, count, done, max_new, eos, n_eos,
                                   None, None, None, st)

    assert call() == 0
    torch.cuda.synchronize()
    assert call(V=409600) == 0
    torch.cuda.synchronize()
    for kw in (dict(B=0), dict(V=0), dict(V=409601), dict(ld=999), dict(logits=None), dict(logits=ctypes.c_void_p(l.data_ptr() + 2)),
               dict(temp=None), dict(top=None), dict(offset=None), dict(n_eos=9), dict(tokens=P(tok)),
               dict(tokens=P(tok), count=P(tok), done=None, max_new=4), dict(ids=P(off), stride=0)):
        assert call(**kw) == MPIG_EINVAL, kw


def test_occupancy_one_wave_at_b32(cuda_lib):
    """At V = 128 256 one cluster of 8 CTAs per row; the device keeps at least 32 such clusters resident (B = 32 in one wave)."""
    n = ctypes.c_int(0)
    assert cuda_lib.mpig_aux_sample_occupancy(128256, ctypes.byref(n)) == 0
    assert n.value >= 32, n.value


# ---- LlamaDecodeRunner.generate -------------------------------------------------------------------------------------------------
GEN_BUF = 16


def _runner(B=2, contexts=None, shared_spill=False):
    from magicpig_b200.llama_runner import LlamaDecodeRunner, LlamaShape
    shape = LlamaShape("tiny", 3, 512, 1024, 4, 2, 1000, 500000.0, 1e-5)   # d = 128, layer 0 dense, vocabulary 1 000
    return LlamaDecodeRunner(shape, 6, 16, B, 512, device=DEV, seed=3, generation_buffer=GEN_BUF, dense_layers=(0,), fused=False,
                             num_contexts=contexts, shared_spill=shared_spill)


def _ids(n, seed):
    return torch.randint(0, 1000, (n,), generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)


def _eager(run, prompts, n_new, T, p, seed):
    """generate() by hand: prefill, then sample() and step() eagerly with manual spills."""
    srv = run.server
    if isinstance(prompts, torch.Tensor):
        run.prefill(prompts) if srv.ctx.num_contexts < run.B else [run.prefill(prompts, request=b) for b in range(run.B)]
    else:
        for b, pr in enumerate(prompts):
            run.prefill(pr, request=b)
    tokens, count, done = run._gen_record()
    count.zero_()
    done.zero_()
    run.set_sampling(T, p, seed=seed, offset=0)
    run.sample()
    used = 0
    for _ in range(n_new - 1):
        if used == GEN_BUF:
            srv.spill_window()
            used = 0
        run.step()
        run.sample()
        used += 1
    n = count.tolist()
    return [tokens[b, :n[b]].tolist() for b in range(run.B)]


@pytest.mark.parametrize("T,p", [(0.0, 0.9), (0.8, 0.9), (1.0, 1.0)])
def test_generate_equals_eager_loop(cuda_lib, T, p):
    """40 tokens (two spills of the 16-row windows) from two prompts: generate() equals the eager loop bitwise."""
    prompts = [_ids(300, 1), _ids(257, 2)]
    out = _runner().generate(prompts, 40, temperature=T, top_p=p, seed=9, check_every=4)
    ref = _eager(_runner(), prompts, 40, T, p, 9)
    assert out == ref
    assert [len(o) for o in out] == [40, 40]
    assert all(0 <= t < 1000 for o in out for t in o)


def test_generate_stops_at_eos(cuda_lib):
    prompts = [_ids(300, 3), _ids(280, 4)]
    run = _runner()
    greedy = run.generate(prompts, 30, temperature=0.0, seed=1)
    k = next(i for i in range(3, 30) if greedy[0][i] not in greedy[0][:i])
    eos = greedy[0][k]
    out = run.generate(prompts, 30, temperature=0.05, eos_token_ids=[eos], seed=1)   # < 0.1: greedy, as in the reference
    want = [g[:g.index(eos) + 1] if eos in g else g for g in greedy]
    assert out == want and out[0][-1] == eos and len(out[0]) == k + 1


def test_generate_forked_prompt(cuda_lib):
    """One prompt forked over 3 requests that share one context (with shared spill), 36 tokens (two spills): until the first spill
    the requests read the same context and windows, so greedy answers agree bitwise there (after it each request's spilled keys
    sit at its own offsets, and the sums round in another order); greedy and sampled answers equal the eager loop, and sampled
    answers differ between requests."""
    prompt = _ids(300, 5)
    run = _runner(B=3, contexts=1, shared_spill=True)
    greedy = run.generate(prompt, 36, temperature=0.0)
    assert [len(g) for g in greedy] == [36] * 3
    assert greedy[0][:GEN_BUF + 1] == greedy[1][:GEN_BUF + 1] == greedy[2][:GEN_BUF + 1]
    assert greedy == _eager(_runner(B=3, contexts=1, shared_spill=True), prompt, 36, 0.0, 0.9, 0)
    sampled = run.generate(prompt, 36, temperature=1.0, top_p=1.0, seed=4)
    assert len({tuple(s) for s in sampled}) > 1
    assert sampled == _eager(_runner(B=3, contexts=1, shared_spill=True), prompt, 36, 1.0, 1.0, 4)


def test_generate_refuses_too_long(cuda_lib):
    run = _runner()
    with pytest.raises(ValueError):
        run.generate(_ids(480, 6), 40)   # 480 + 40 > 512
    assert run._gen_graph is None and run.pos.tolist() == [0, 0]
