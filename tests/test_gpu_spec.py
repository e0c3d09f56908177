"""Speculative decoding on the device: mpig_aux_verify_sample and mpig_aux_ngram_draft (csrc/aux_sample.cu) against the restatements
in tests/support/spec_rule.py, chi-square tests of the emitted tokens' law, and LlamaDecodeRunner.generate(draft_tokens=k) against
an eager loop of the same calls."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

from magicpig_b200 import _native as N
from magicpig_b200.ops import ngram_draft, sample, verify_sample
from tests.support import sample_rule as R
from tests.support import spec_rule as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MPIG_EINVAL = -1   # include/magicpig_b200.h
TEMPS = (0.0, 0.6, 1.0, 0.6, 1.5)
TOPS = (0.9, 0.9, 1.0, 0.5, 0.95)
REGIMES = ("flat", "peaked", "ties", "masked")


def _rows(regime, n, V, g):
    if regime == "flat":
        l = torch.randn((n, V), generator=g) * 0.05
    elif regime == "peaked":
        l = torch.randn((n, V), generator=g)
        for r in range(n):
            l[r, torch.randint(0, V, (1 + r % 3,), generator=g)] = 25.0 + torch.rand(1 + r % 3, generator=g)
    elif regime == "ties":
        l = torch.round(torch.randn((n, V), generator=g) * 1.5)
    else:
        l = torch.randn((n, V), generator=g) * 2
        l[torch.rand((n, V), generator=g) < 0.9] = float("-inf")
    return l.float()


def _draft_for(row, case, p):
    """A draft that exercises `case` on this row: the argmax, a kept token, the boundary, a token outside the nucleus, a -inf token."""
    l = row.double()
    order = torch.argsort(-l, stable=True)
    w = torch.softmax(l, 0)
    n_keep = int((torch.cumsum(w[order], 0) - w[order] <= p).sum())
    finite = int(torch.isfinite(l).sum())
    pick = [0, max(0, n_keep // 2), max(0, n_keep - 1), min(finite - 1, n_keep), l.numel() - 1][case % 5]
    return int(order[pick])


def _case(V, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    logits = torch.stack([_rows(REGIMES[(b + seed) % 4], T, V, g) for b in range(B)])   # (B, T, V)
    temp = torch.tensor([TEMPS[b % 5] for b in range(B)], dtype=torch.float32)
    top = torch.tensor([TOPS[(b // 5 + b) % 5] for b in range(B)], dtype=torch.float32)
    ids = torch.zeros((B, 8), dtype=torch.int64)
    for b in range(B):
        ids[b, 0] = b
        for t in range(T - 1):
            ids[b, t + 1] = _draft_for(logits[b, t], b + t, float(top[b]))
    return logits, temp, top, ids


def _book(B, seed):
    g = torch.Generator().manual_seed(seed)
    length = torch.randint(0, 6, (B,), generator=g, dtype=torch.int32)
    limit = length + torch.randint(1, 9, (B,), generator=g, dtype=torch.int32)
    done = (torch.rand(B, generator=g) < 0.15).int()
    return length, limit, done


def _verify(logits, temp, top, ids, seed, off, book=None, eos=()):
    B, T, V = logits.shape
    i32 = lambda x: x.to(DEV, torch.int32).contiguous()  # noqa: E731
    out = dict(ids=ids.to(DEV).clone(), drop=torch.full((B,), -7, dtype=torch.int32, device=DEV),
               debug=torch.zeros((B, T, 9), dtype=torch.int64, device=DEV), debug_w=torch.full((B, T, V), -1.0, device=DEV),
               status=torch.zeros(((B + 31) // 32,), dtype=torch.int32, device=DEV),
               steps=torch.zeros(B, dtype=torch.int32, device=DEV), accepted=torch.zeros(B, dtype=torch.int32, device=DEV))
    if book is None:   # every request running, room for every token
        book = (torch.zeros(B, dtype=torch.int32), torch.full((B,), 24, dtype=torch.int32), torch.zeros(B, dtype=torch.int32))
    length, limit, done = book
    out.update(history=torch.full((B, 24), -1, dtype=torch.int32, device=DEV), length=i32(length), limit=i32(limit), done=i32(done))
    offset = torch.tensor([off], dtype=torch.int64, device=DEV)
    verify_sample(logits.to(DEV), temp.to(DEV), top.to(DEV), seed, offset, out["ids"], drop=out["drop"], history=out["history"],
                  length=out["length"], limit=out["limit"], done=out["done"], steps=out["steps"], accepted=out["accepted"],
                  eos_token_ids=eos, status=out["status"], debug=out["debug"], debug_w=out["debug_w"])
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


@pytest.mark.parametrize("V", [128256, 32000])
@pytest.mark.parametrize("B", [1, 8, 32])
@pytest.mark.parametrize("T", [1, 2, 4, 8])
def test_exact_against_restatement(cuda_lib, V, B, T):
    """Each row's debug integers and weights equal mpig_aux_sample's on the same row bitwise; tokens, drop, history, counters and
    done equal the restatement on the kernel's own weights bitwise; at T = 1 the token is mpig_aux_sample's."""
    seed = V + 10 * B + T
    logits, temp, top, ids = _case(V, B, T, seed)
    book = _book(B, seed)
    eos = (int(ids[0, 1]),) if T > 1 else ()
    out = _verify(logits, temp, top, ids, 1234, 77, book, eos)
    for t in range(T):
        sdbg = torch.zeros((B, 5), dtype=torch.int64, device=DEV)
        sw = torch.full((B, V), -1.0, device=DEV)
        tok = sample(logits[:, t].to(DEV), temp.to(DEV), top.to(DEV), 1234, torch.tensor([77], device=DEV), debug=sdbg, debug_w=sw)
        assert torch.equal(out["debug"][:, t, :5], sdbg.cpu()), f"row {t}: debug differs from mpig_aux_sample"
        assert torch.equal(out["debug_w"][:, t], sw.cpu()), f"row {t}: weights differ from mpig_aux_sample"
        if T == 1:
            assert torch.equal(out["ids"][:, 0], tok.cpu())
    length, limit, done = book
    for b in range(B):
        W_rows = [R.fixed_point(out["debug_w"][b, t].double().numpy()) for t in range(T)]
        want = S.request(logits[b].numpy(), float(temp[b]), float(top[b]), 1234, 77, b, ids[b].tolist(), W_rows=W_rows,
                         done=bool(done[b]), length=int(length[b]), limit=int(limit[b]), eos=eos)
        assert [tuple(r[3]) for r in want["rows"]] == [tuple(x) for x in out["debug"][b].tolist()], f"request {b}: debug"
        assert int(out["ids"][b, 0]) == want["final"] and int(out["drop"][b]) == want["drop"], f"request {b}"
        n0 = int(length[b])
        assert out["history"][b, n0:n0 + len(want["emitted"])].tolist() == want["emitted"]
        assert int(out["length"][b]) == want["length"] and int(out["done"][b]) == int(want["done"])
        assert int(out["steps"][b]) == int(want["counted"]) and int(out["accepted"][b]) == (want["k"] if want["counted"] else 0)
        assert out["ids"][b, 1:].tolist() == ids[b, 1:].tolist()   # the drafts are read, never written
    assert not out["status"].any()


def _chi2(counts, probs):
    keep = probs > 0
    assert counts[~keep].sum() == 0
    return stats.chisquare(counts[keep], probs[keep] / probs[keep].sum() * counts[keep].sum()).pvalue


def _nucleus(l, T, p):
    W = R.fixed_point(R.weights_fp64(l, T))
    keep = R.keep_mask(W, R.nucleus_threshold(p, int(W.sum())))
    q = np.where(keep, W, 0).astype(np.float64)
    return q / q.sum(), keep


@pytest.mark.parametrize("likely", [True, False])
def test_chi_square(cuda_lib, likely):
    """T = 2 over 200 000 (offset, request) draws: the first token follows row 0's nucleus, acceptance happens with p(d), and the
    second token given acceptance follows row 1's nucleus.  The residual without excluding d, and the un-truncated distribution,
    are rejected."""
    V, Bq, n_off, Tt, p = 200, 2000, 100, 0.8, 0.9
    g = torch.Generator().manual_seed(5)
    rows = torch.randn((2, V), generator=g) * 1.5
    q0, keep0 = _nucleus(rows[0].numpy(), Tt, p)
    q1, _ = _nucleus(rows[1].numpy(), Tt, p)
    order = np.argsort(-q0, kind="stable")
    d = int(order[0]) if likely else int(order[int(keep0.sum()) - 1])
    logits = rows[None].expand(Bq, 2, V).contiguous().to(DEV)
    temp, top = torch.full((Bq,), Tt, device=DEV), torch.full((Bq,), p, device=DEV)
    ids = torch.zeros((Bq, 2), dtype=torch.int64, device=DEV)
    hist = torch.zeros((Bq, 2), dtype=torch.int32, device=DEV)
    length, limit, done = (torch.zeros(Bq, dtype=torch.int32, device=DEV), torch.full((Bq,), 2, dtype=torch.int32, device=DEV),
                           torch.zeros(Bq, dtype=torch.int32, device=DEV))
    offset = torch.zeros(1, dtype=torch.int64, device=DEV)
    first, acc, second = np.zeros(V), 0, np.zeros(V)
    for o in range(n_off):
        ids[:, 1] = d
        length.zero_()
        done.zero_()
        offset.fill_(o)
        verify_sample(logits, temp, top, 99, offset, ids, history=hist, length=length, limit=limit, done=done)
        h, n = hist.cpu().numpy(), length.cpu().numpy()
        first += np.bincount(h[:, 0], minlength=V)
        a = n == 2
        acc += int(a.sum())
        second += np.bincount(h[a, 1], minlength=V)
    N_ = Bq * n_off
    assert _chi2(first, q0) > 1e-3
    assert stats.binomtest(acc, N_, q0[d]).pvalue > 1e-3
    assert _chi2(second, q1) > 1e-3
    no_excl = q0 * (1 - q0[d])
    no_excl[d] += q0[d]
    assert stats.chisquare(first[q0 > 0], no_excl[q0 > 0] / no_excl[q0 > 0].sum() * first.sum()).pvalue < 1e-6 or not likely
    full = np.exp((rows[0].double().numpy() - rows[0].max().item()) / Tt)
    full /= full.sum()
    assert stats.chisquare(first, full * first.sum()).pvalue < 1e-6
    if likely:   # the residual law without excluding d puts q0[d]^2 extra on d: visible when q0[d] is large
        assert q0[d] > 0.05


def test_full_acceptance_and_eos(cuda_lib):
    """Greedy rows with drafts equal to the argmax chain accept all T - 1; an EOS id among them ends the request there."""
    B, T, V = 4, 8, 1000
    g = torch.Generator().manual_seed(8)
    logits = torch.randn((B, T, V), generator=g)
    am = logits.argmax(-1)
    ids = torch.zeros((B, 8), dtype=torch.int64)
    ids[:, 1:T] = am[:, :T - 1]
    temp, top = torch.zeros(B), torch.ones(B)
    out = _verify(logits, temp, top, ids, 1, 0, (torch.zeros(B, dtype=torch.int32), torch.full((B,), 20, dtype=torch.int32),
                                                  torch.zeros(B, dtype=torch.int32)))
    assert out["drop"].tolist() == [0] * B and out["accepted"].tolist() == [T - 1] * B
    assert out["ids"][:, 0].tolist() == am[:, T - 1].tolist()
    assert torch.equal(out["history"][:, :T], am.int())
    eos = int(am[2, 3])
    out = _verify(logits, temp, top, ids, 1, 0, (torch.zeros(B, dtype=torch.int32), torch.full((B,), 20, dtype=torch.int32),
                                                 torch.zeros(B, dtype=torch.int32)), eos=(eos,))
    assert out["done"][2] == 1 and out["history"][2, :5].tolist() == am[2, :4].tolist() + [-1] and out["length"][2] == 4
    # limit inside the drafts, and a request already done
    out = _verify(logits, temp, top, ids, 1, 0, (torch.tensor([0, 0, 5, 0], dtype=torch.int32), torch.tensor([3, 20, 20, 20],
                                                 dtype=torch.int32), torch.tensor([0, 1, 0, 0], dtype=torch.int32)))
    assert out["length"].tolist()[:2] == [3, 0] and out["done"].tolist()[:2] == [1, 1]
    assert out["drop"][1] == T and out["steps"][1] == 0 and (out["history"][1] == -1).all()


def test_invalid_rows_set_status(cuda_lib):
    B, T, V = 3, 4, 500
    g = torch.Generator().manual_seed(9)
    logits = torch.randn((B, T, V), generator=g)
    am = logits.argmax(-1)
    ids = torch.zeros((B, 8), dtype=torch.int64)
    ids[:, 1:T] = am[:, :T - 1]
    logits[0, 0, 7] = float("nan")           # row 0 invalid: k = 0, token 0, status
    logits[1, 2, :] = float("-inf")          # row 2 invalid after two accepted drafts
    logits[2, 3, 3] = float("inf")           # row 3 invalid, but row 1 rejects first
    ids[2, 2] = (am[2, 1] + 1) % V
    out = _verify(logits, torch.zeros(B), torch.ones(B), ids, 1, 0)
    assert out["ids"][:, 0].tolist()[:2] == [0, 0] and out["drop"].tolist() == [3, 1, 2]
    assert out["status"].tolist() == [0b011]


def test_refusals(cuda_lib):
    lib = N.load()
    x = torch.zeros((2, 2, 64), device=DEV)
    ids = torch.zeros((2, 8), dtype=torch.int64, device=DEV)
    rows = torch.zeros((2, 8, 2), dtype=torch.int32, device=DEV)
    tp = torch.ones(2, device=DEV)
    off = torch.zeros(1, dtype=torch.int64, device=DEV)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    eos = (ctypes.c_int32 * 9)(*range(9))

    def call(T=2, logits=P(x), ld_b=128, ld_t=64, n_eos=0, ids_p=P(ids), stride=8):
        return lib.mpig_aux_verify_sample(logits, 2, T, 64, ld_b, ld_t, P(tp), P(tp), 0, P(off), ids_p, stride, P(rows), None, None, 0,
                                          None, None, None, None, None, eos, n_eos, None, None, None, None)
    assert call() == 0
    torch.cuda.synchronize()
    for kw in (dict(T=0), dict(T=9, ld_b=9 * 64), dict(ld_t=32), dict(ld_b=100), dict(n_eos=9), dict(ids_p=None),
               dict(logits=ctypes.c_void_p(x.data_ptr() + 2)), dict(ids_p=ctypes.c_void_p(ids.data_ptr() + 4)), dict(stride=1)):
        assert call(**kw) == MPIG_EINVAL, kw
    h = torch.zeros((2, 16), dtype=torch.int32, device=DEV)
    n = torch.zeros(2, dtype=torch.int32, device=DEV)
    for T, gmin, gmax in ((0, 1, 3), (9, 1, 3), (4, 0, 3), (4, 1, 9), (4, 3, 2)):
        assert lib.mpig_aux_ngram_draft(P(h), 2, 16, P(n), P(ids), 8, T, gmin, gmax, None) == MPIG_EINVAL


def test_capture_and_determinism(cuda_lib):
    B, T, V = 8, 4, 32000
    logits, temp, top, ids0 = _case(V, B, T, 3)
    logits, temp, top = logits.to(DEV), temp.to(DEV), top.to(DEV)
    hist = torch.randint(0, 50, (B, 300), dtype=torch.int32, device=DEV)
    length = torch.full((B,), 200, dtype=torch.int32, device=DEV)
    limit = torch.full((B,), 300, dtype=torch.int32, device=DEV)
    done = torch.zeros(B, dtype=torch.int32, device=DEV)
    off = torch.zeros(1, dtype=torch.int64, device=DEV)
    ids, drop = torch.zeros((B, 8), dtype=torch.int64, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV)

    def body():
        ngram_draft(hist, length, ids, T)
        verify_sample(logits, temp, top, 5, off, ids, drop=drop, history=hist, length=length, limit=limit, done=done)
        off.add_(1)

    state = lambda: [x.clone() for x in (hist, length, done, ids, drop, off)]  # noqa: E731
    start = state()
    for _ in range(3):
        body()
    eager = state()
    for x, y in zip((hist, length, done, ids, drop, off), start):
        x.copy_(y)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        body()
    torch.cuda.current_stream().wait_stream(s)
    for x, y in zip((hist, length, done, ids, drop, off), start):
        x.copy_(y)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()
    for x, y in zip((hist, length, done, ids, drop, off), start):
        x.copy_(y)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(state(), eager))


# ---- prompt lookup ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,n_max,T,gmin,gmax", [(8, 99024, 8, 1, 3), (8, 5000, 4, 2, 8), (32, 700, 8, 1, 3), (3, 40, 2, 1, 1)])
def test_ngram_against_restatement(cuda_lib, B, n_max, T, gmin, gmax):
    """Random histories with planted repeats (copies of earlier spans, a periodic tail on some), ragged lengths up to n_max."""
    g = np.random.default_rng(n_max + B)
    ld = n_max + 16
    hist = g.integers(0, 3000, (B, ld)).astype(np.int32)
    lengths = [n_max] + [int(x) for x in g.integers(0, n_max + 1, B - 1)]
    lengths[-1] = min(lengths[-1], 1)
    for b in range(B):
        n = lengths[b]
        for _ in range(4):   # copies of earlier spans
            if n > 40:
                a, c = sorted(g.integers(0, n - 10, 2))
                L = int(g.integers(1, 10))
                hist[b, c:c + L] = hist[b, a:a + L]
        if b % 3 == 1 and n > 20:
            hist[b, n - 12:n] = np.tile(hist[b, n - 15:n - 12], 4)   # a period of 3 at the end
        if b % 4 == 2 and n > 10:
            hist[b, n - 1] = 99999   # no match
    h = torch.from_numpy(hist).to(DEV)
    ln = torch.tensor(lengths, dtype=torch.int32, device=DEV)
    ids = torch.full((B, 8), -5, dtype=torch.int64, device=DEV)
    ngram_draft(h, ln, ids, T, gmin, gmax)
    torch.cuda.synchronize()
    got = ids.cpu()
    for b in range(B):
        want = S.ngram_drafts(hist[b, :lengths[b]], T, gmin, gmax)
        assert got[b, 1:T].tolist() == want, f"request {b} (n = {lengths[b]})"
        assert got[b, 0] == -5 and (got[b, T:] == -5).all()


# ---- generate(draft_tokens=k) ---------------------------------------------------------------------------------------------------
GEN_BUF = 16


def _runner(B=2, contexts=None, shared_spill=False):
    from magicpig_b200.llama_runner import LlamaDecodeRunner, LlamaShape
    shape = LlamaShape("tiny", 3, 512, 1024, 4, 2, 1000, 500000.0, 1e-5)   # d = 128, layer 0 dense, vocabulary 1 000
    return LlamaDecodeRunner(shape, 6, 16, B, 512, device=DEV, seed=3, generation_buffer=GEN_BUF, dense_layers=(0,), fused=False,
                             num_contexts=contexts, shared_spill=shared_spill, max_query_tokens=8)


def _ids(n, seed, period=0):
    x = torch.randint(0, 1000, (n,), generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)
    if period:   # text that repeats itself, so prompt lookup finds matches
        x = x[:period].repeat(n // period + 1)[:n]
    return x


def _eager_spec(run, prompts, n_new, temp, top_p, seed, k, ngram=(1, 3)):
    """generate(draft_tokens=k) by hand: the same calls eagerly, each step checked against the restatement on its own logits."""
    from magicpig_b200.llama_runner import spec_spill_every
    srv, B, T = run.server, run.B, k + 1
    if isinstance(prompts, torch.Tensor):
        prompts = [prompts] * B
        run.prefill(prompts[0]) if srv.ctx.num_contexts < B else [run.prefill(prompts[0], request=b) for b in range(B)]
    else:
        for b, pr in enumerate(prompts):
            run.prefill(pr, request=b)
    hist, length, limit, done = run._history()
    P = [int(p.numel()) for p in prompts]
    for b in range(B):
        hist[b, :P[b]] = prompts[b].int()
    length.copy_(torch.tensor(P, dtype=torch.int32))
    limit.copy_(torch.tensor([x + n_new for x in P], dtype=torch.int32))
    done.zero_()
    run.set_sampling(temp, top_p, seed=seed, offset=0)
    eos = run.eos_token_ids
    args = lambda: (run.temperature, run.top_p, seed, run.sample_offset, run.ids_tok)  # noqa: E731
    verify_sample(run.logits[:, None], *args(), drop=run._spec_drop, history=hist, length=length, limit=limit, done=done,
                  eos_token_ids=eos)
    run.sample_offset.add_(1)
    every, since = spec_spill_every(GEN_BUF, k), 0
    temps, tops = run.temperature.tolist(), run.top_p.tolist()
    for _ in range(n_new - 1):
        if since == every:
            srv.spill_window()
            since = 0
        ngram_draft(hist, length, run.ids_tok, T, *ngram)
        logits = run.step_tokens(T)
        before = (logits.cpu().numpy().copy(), run.ids_tok[:, :T].cpu().tolist(), length.tolist(), done.tolist(), int(run.sample_offset))
        dw = torch.zeros((B, T, logits.shape[2]), device=DEV)
        verify_sample(logits, *args(), drop=run._spec_drop, history=hist, length=length, limit=limit, done=done, eos_token_ids=eos,
                      debug_w=dw)
        lg, idr, n0, d0, off = before
        h = hist.cpu()
        for b in range(B):
            W_rows = [R.fixed_point(dw[b, t].double().cpu().numpy()) for t in range(T)]
            want = S.request(lg[b], temps[b], tops[b], seed, off, b, idr[b], W_rows=W_rows, done=bool(d0[b]), length=n0[b],
                             limit=int(limit[b]), eos=eos)
            assert h[b, n0[b]:n0[b] + len(want["emitted"])].tolist() == want["emitted"]
            assert int(run._spec_drop[b]) == want["drop"] and int(run.ids_tok[b, 0]) == want["final"]
            if temps[b] == 0:   # greedy: every emitted token is the argmax of the row that produced it
                assert want["emitted"] == [int(np.argmax(lg[b, t])) for t in range(len(want["emitted"]))]
        srv.rewind(run._spec_drop)
        run.pos.sub_(run._spec_drop.long())
        run.sample_offset.add_(1)
        since += 1
    n = length.tolist()
    return [hist[b, P[b]:n[b]].tolist() for b in range(B)]


@pytest.mark.parametrize("k", [1, 3, 7])
@pytest.mark.parametrize("temp,top_p", [(0.0, 0.9), (0.6, 0.9)])
def test_generate_equals_eager_loop(cuda_lib, k, temp, top_p):
    """40 tokens from two prompts that repeat themselves (several spills of the 16-row windows): generate(draft_tokens=k) equals the
    eager loop bitwise, and each eager step equals the restatement."""
    prompts = [_ids(300, 1, period=37), _ids(257, 2, period=11)]
    run = _runner()
    out = run.generate(prompts, 40, temperature=temp, top_p=top_p, seed=9, check_every=4, draft_tokens=k)
    ref = _eager_spec(_runner(), prompts, 40, temp, top_p, 9, k)
    assert out == ref
    assert [len(o) for o in out] == [40, 40]
    st = run.last_generate_stats
    assert st["draft_tokens"] == k and 1.0 <= st["tokens_per_step"] <= k + 1
    assert all(1 <= s <= 39 for s in st["steps"]) and all(0 <= a <= k * s for a, s in zip(st["accepted"], st["steps"]))
    if temp == 0:   # drafts from the text the greedy model repeats are accepted: partial rewinds and multi-token appends run
        assert sum(st["accepted"]) > 0, st
    _assert_rows_match_tokens(run, [300, 257], out)


def _assert_rows_match_tokens(run, P, out):
    """Every request holds the prompt and its emitted tokens but the last, whether it ended early or not, and no capacity flag."""
    assert run.pos.tolist() == [p + len(o) - 2 for p, o in zip(P, out)]
    assert run.server.ctx.error_flags() == 0


def test_generate_at_the_capacity_bounds(cuda_lib):
    """P + max_new_tokens + k = max_length for request 0 and an EOS that ends request 1 early, greedy with accepted drafts: the
    requests that end (at their limit or an EOS, possibly inside the accepted drafts) keep only their emitted tokens' rows, and
    the replays after they end stay inside the caches.  The same with dense_tail_rows = max_new_tokens + k over a forked prompt."""
    k, n = 3, 40
    prompts = [_ids(512 - n - k, 1, period=37), _ids(257, 2, period=11)]
    ref = _runner().generate(prompts, n, temperature=0.0, draft_tokens=k)
    eos = ref[1][12]
    run = _runner()
    out = run.generate(prompts, n, temperature=0.0, draft_tokens=k, eos_token_ids=[eos], check_every=64)
    assert out[0] == (ref[0][:ref[0].index(eos) + 1] if eos in ref[0] else ref[0])
    assert out[1] == ref[1][:ref[1].index(eos) + 1] and len(out[1]) <= 13
    assert sum(run.last_generate_stats["accepted"]) > 0
    _assert_rows_match_tokens(run, [int(p.numel()) for p in prompts], out)

    from magicpig_b200.llama_runner import LlamaDecodeRunner, LlamaShape
    shape = LlamaShape("tiny", 3, 512, 1024, 4, 2, 1000, 500000.0, 1e-5)
    run = LlamaDecodeRunner(shape, 6, 16, 3, 512, device=DEV, seed=3, generation_buffer=GEN_BUF, dense_layers=(0,), fused=False,
                            num_contexts=1, shared_spill=True, max_query_tokens=8, dense_tail_rows=n + k)
    prompt = _ids(300, 5, period=23)
    out = run.generate(prompt, n, temperature=0.6, top_p=0.9, seed=4, draft_tokens=k, check_every=64)
    assert [len(o) for o in out] == [n] * 3
    _assert_rows_match_tokens(run, [300] * 3, out)


def test_generate_forked_prompt(cuda_lib):
    """One prompt forked over 3 requests sharing one context with shared spill, sampled, k = 3: equals the eager loop."""
    prompt = _ids(300, 5, period=23)
    run = _runner(B=3, contexts=1, shared_spill=True)
    out = run.generate(prompt, 36, temperature=0.6, top_p=0.9, seed=4, draft_tokens=3)
    assert out == _eager_spec(_runner(B=3, contexts=1, shared_spill=True), prompt, 36, 0.6, 0.9, 4, 3)
    assert len({tuple(o) for o in out}) > 1


def test_caller_drafts_argmax_chain(cuda_lib):
    """draft=None: the caller's drafts in ids_tok[:, 1:T]; drafts equal to the greedy chain of the verification logits are all
    accepted."""
    prompts = [_ids(300, 1), _ids(257, 2)]
    T = 4
    run = _runner()
    run.generate(prompts, 2, temperature=0.0, draft_tokens=T - 1)   # prefill, the history and the first token
    hist, length, _, done = run._history()
    done.zero_()
    run.history_limit.fill_(500)
    # probe: one eager step with arbitrary drafts, rolled back, gives the row-0 argmax; repeat to build the chain
    chain = []
    for t in range(T - 1):
        run.ids_tok[:, 1:T] = torch.tensor([chain + [0] * (T - 1 - len(chain))] * 2, device=DEV)
        n0 = length.clone()
        logits = run.step_tokens(T)
        chain.append(int(logits[0, t].argmax()))
        run.server.rewind(torch.full((2,), T, dtype=torch.int32, device=DEV))
        run.pos.sub_(T)
        length.copy_(n0)
    run.ids_tok[0, 1:T] = torch.tensor(chain, device=DEV)
    acc0 = run.spec_accepted.clone()
    run.spec_step(T, draft=None)
    torch.cuda.synchronize()
    assert int(run.spec_accepted[0] - acc0[0]) == T - 1 and int(run._spec_drop[0]) == 0


def test_generate_refusals(cuda_lib):
    run = _runner()
    p = _ids(300, 1)
    for kw in (dict(draft_tokens=8), dict(draft_tokens=16), dict(ngram=(0, 3)), dict(ngram=(1, 9))):
        with pytest.raises(ValueError):
            run.generate(p, 20, draft_tokens=kw.pop("draft_tokens", 3), **kw)
    with pytest.raises(ValueError):
        run.generate(_ids(470, 2), 40, draft_tokens=3)   # 470 + 40 + 3 > 512
    assert run._spec_graph is None and run.token_history is None and run.pos.tolist() == [0, 0]
