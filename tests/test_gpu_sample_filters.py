"""Sampling filters on the device: mpig_aux_sample_filtered and mpig_aux_verify_sample_filtered (csrc/aux_sample.cu) against the
unfiltered calls with neutral filters and against the restatement in tests/support/filter_rule.py, chi-square tests of the
filtered law, the penalty table's bookkeeping, capture, and LlamaDecodeRunner.generate() with filters against an eager loop."""
import numpy as np
import pytest
import torch
from scipy import stats

from magicpig_b200 import ops
from magicpig_b200.ops import SampleFilters, sample, verify_sample
from tests.support import filter_rule as F
from tests.support import sample_rule as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
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


def _filters(B, V, seed, neutral=False, ld_extra=3):
    """Per-request values cycling through top_k {0, 1, 2, 50, V + 1}, min_p {0, 0.05, 1} and mixed penalties; a table with prompt
    bits and counts."""
    g = torch.Generator().manual_seed(seed)
    f = SampleFilters.neutral(B, V, "cpu")
    f.table = torch.zeros((B, V + ld_extra), dtype=torch.int32)
    if neutral:
        return f
    f.top_k = torch.tensor([(0, 1, 2, 50, V + 1)[(b + seed) % 5] for b in range(B)], dtype=torch.int32)
    f.min_p = torch.tensor([(0.0, 0.05, 1.0, 0.0)[(b + seed) % 4] for b in range(B)])
    f.repetition_penalty = torch.tensor([(1.0, 1.3, 0.7)[(b + seed) % 3] for b in range(B)])
    f.presence_penalty = torch.tensor([(0.0, 0.5, -1.0)[(b + 2 * seed) % 3] for b in range(B)])
    f.frequency_penalty = torch.tensor([(0.0, 0.3, -0.2, 2.0)[(b + seed) % 4] for b in range(B)])
    for b in range(B):
        f.table[b, torch.randint(0, V, (200,), generator=g)] = ops.PROMPT_BIT
        f.table[b, torch.randint(0, V, (100,), generator=g)] += torch.randint(1, 5, (100,), generator=g, dtype=torch.int32)
    return f


def _to(f, dev=DEV):
    return SampleFilters(*(getattr(f, k).to(dev) for k in ("top_k", "min_p", "repetition_penalty", "presence_penalty",
                                                           "frequency_penalty", "table")))


def _vals(f, b):
    return F.device_values(int(f.top_k[b]), float(f.min_p[b]), float(f.repetition_penalty[b]), float(f.presence_penalty[b]),
                           float(f.frequency_penalty[b]))


def _table_row(f, b, V):
    return f.table[b, :V].numpy().astype(np.int64) & 0xFFFFFFFF


def _case(V, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    logits = torch.stack([_rows(REGIMES[(b + seed) % 4], T, V, g) for b in range(B)])
    temp = torch.tensor([TEMPS[b % 5] for b in range(B)], dtype=torch.float32)
    top = torch.tensor([TOPS[(b // 5 + b) % 5] for b in range(B)], dtype=torch.float32)
    ids = torch.zeros((B, 8), dtype=torch.int64)
    for b in range(B):
        ids[b, 0] = b
        for t in range(T - 1):   # the row's argmax, a repeat of an earlier draft, or a random token
            ids[b, t + 1] = [int(logits[b, t].argmax()), int(ids[b, max(t, 1)]), int(torch.randint(0, V, (1,), generator=g))][(b + t) % 3]
    return logits, temp, top, ids


@pytest.mark.parametrize("V", [128256, 32000])
@pytest.mark.parametrize("B", [1, 8, 32])
def test_neutral_filters_equal_unfiltered(cuda_lib, V, B):
    """Neutral filters: token, debug integers and weights of both calls equal the unfiltered calls' bit for bit."""
    T = 4
    logits, temp, top, ids = _case(V, B, T, V + B)
    lg, tp, pp = logits.to(DEV), temp.to(DEV), top.to(DEV)
    f = _to(_filters(B, V, 1, neutral=True))
    off = torch.tensor([5], device=DEV)
    out = {}
    for filt in (None, f):
        n = 5 if filt is None else 8
        dbg, dw = torch.zeros((B, n), dtype=torch.int64, device=DEV), torch.zeros((B, V), device=DEV)
        tok = sample(lg[:, 0], tp, pp, 11, off, debug=dbg, debug_w=dw, filters=filt)
        vd, vw = torch.zeros((B, T, n + 4), dtype=torch.int64, device=DEV), torch.zeros((B, T, V), device=DEV)
        vid, drop = ids.to(DEV), torch.zeros(B, dtype=torch.int32, device=DEV)
        verify_sample(lg, tp, pp, 11, off, vid, drop=drop, debug=vd, debug_w=vw, filters=filt)
        out[filt is None] = (tok.cpu(), dbg[:, :5].cpu(), dw.cpu(), vd[..., :9].cpu(), vw.cpu(), vid.cpu(), drop.cpu())
    for a, b in zip(out[True], out[False]):
        assert torch.equal(a, b)
    assert not f.table.any()


@pytest.mark.parametrize("V", [128256, 32000])
@pytest.mark.parametrize("B", [1, 8, 32])
@pytest.mark.parametrize("T", [1, 2, 4, 8])
def test_exact_against_restatement(cuda_lib, V, B, T):
    """Tokens, debug integers, drop, history and the table equal the restatement on the kernel's own weights bit for bit; the
    weights are those of the restated penalised logits within the fp32 bound of fp64; sample_filtered is verify row 0 at T = 1."""
    seed = V + 10 * B + T
    logits, temp, top, ids = _case(V, B, T, seed)
    fh = _filters(B, V, seed)
    f = _to(fh)
    off = torch.tensor([77], device=DEV)
    vid = ids.to(DEV)
    dbg, dw = torch.zeros((B, T, 12), dtype=torch.int64, device=DEV), torch.zeros((B, T, V), device=DEV)
    hist = torch.full((B, 24), -1, dtype=torch.int32, device=DEV)
    length, limit = torch.zeros(B, dtype=torch.int32, device=DEV), torch.full((B,), 24, dtype=torch.int32, device=DEV)
    done, drop = torch.zeros(B, dtype=torch.int32, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV)
    verify_sample(logits.to(DEV), temp.to(DEV), top.to(DEV), 1234, off, vid, drop=drop, history=hist, length=length, limit=limit,
                  done=done, debug=dbg, debug_w=dw, filters=f)
    torch.cuda.synchronize()
    dbg, dw, vid, tab = dbg.cpu(), dw.cpu(), vid.cpu(), f.table.cpu()
    for b in range(B):
        vals, trow = _vals(fh, b), _table_row(fh, b, V)
        W_rows = [R.fixed_point(dw[b, t].double().numpy()) for t in range(T)]
        want = F.request(logits[b].numpy(), float(temp[b]), float(top[b]), vals, trow, 1234, 77, b, ids[b].tolist(), W_rows=W_rows,
                         length=0, limit=24)
        assert [tuple(r[3]) for r in want["rows"]] == [tuple(x) for x in dbg[b].tolist()], f"request {b}: debug"
        assert int(vid[b, 0]) == want["final"] and int(drop[b]) == want["drop"], f"request {b}"
        assert hist[b, :len(want["emitted"])].tolist() == want["emitted"]
        assert (tab[b, :V].numpy().astype(np.int64) & 0xFFFFFFFF).tolist() == want["table"].astype(np.int64).tolist()
        assert tab[b, V:].tolist() == fh.table[b, V:].tolist()
        if float(temp[b]) > 0:
            for t in range(T):   # the kernel's weights against fp64 of the restated penalised logits
                drafts = ids[b, 1:t + 1].tolist()
                l3 = F.penalised(logits[b, t].numpy(), trow, F.draft_counts(drafts, V), vals)
                w64 = R.weights_fp64(l3, float(temp[b]))
                bound = R.weight_rel_bound(l3, float(temp[b])) * w64 + 2.0 ** -40
                assert (np.abs(dw[b, t].double().numpy() - w64) <= bound).all()
    if T == 1:
        sd = torch.zeros((B, 8), dtype=torch.int64, device=DEV)
        f2 = _to(fh)
        tok = sample(logits[:, 0].to(DEV), temp.to(DEV), top.to(DEV), 1234, off, debug=sd, filters=f2)
        sd = sd.cpu()   # (S, thr, S_keep, K, target, n_k, S_k, n_m) against the row's first five and its last three
        assert torch.equal(tok.cpu(), vid[:, 0]) and torch.equal(sd[:, :5], dbg[:, 0, :5]) and torch.equal(sd[:, 5:], dbg[:, 0, 9:])


def test_boundary_ties(cuda_lib):
    """Ties exactly at the top-k and the min-p boundary: the lower indices stay, n_k and n_m as restated."""
    V, B = 32000, 4
    l = torch.full((B, V), -5.0)
    l[:, [10, 20, 30, 40]] = 3.0        # four tied maxima
    l[:, [5, 15, 25]] = 3.0 - 0.6931472  # w = 1/2 exactly in fp32 at T = 1? close; ties among themselves
    fh = SampleFilters.neutral(B, V, "cpu")
    fh.top_k = torch.tensor([2, 5, 0, 6], dtype=torch.int32)
    fh.min_p = torch.tensor([0.0, 0.0, 1.0, 0.3])
    temp, top = torch.ones(B), torch.ones(B)
    dbg = torch.zeros((B, 8), dtype=torch.int64, device=DEV)
    dw = torch.zeros((B, V), device=DEV)
    f = _to(fh)
    for off in range(20):
        tok = sample(l.to(DEV), temp.to(DEV), top.to(DEV), 3, torch.tensor([off], device=DEV), debug=dbg, debug_w=dw, filters=f)
        tok, d, w = tok.cpu(), dbg.cpu(), dw.cpu()
        for b in range(B):
            want = F.sample_row(l[b].numpy(), 1.0, 1.0, _vals(fh, b), np.zeros(V, dtype=np.int64), 3, off, b,
                                W=R.fixed_point(w[b].double().numpy()))
            assert (int(tok[b]), tuple(d[b].tolist())) == want
        assert int(tok[0]) in (10, 20) and int(tok[2]) in (10, 20, 30, 40)
    assert d[0, 3] == 2 and d[2, 3] == 4


def test_out_of_range_device_values_are_neutral(cuda_lib, monkeypatch):
    """Each kind of out-of-range device value behaves as its neutral value (the Python checks are bypassed to reach the device)."""
    monkeypatch.setattr(ops, "check_filter_values", lambda *a, **k: None)
    V, B = 32000, 6
    logits, temp, top, _ = _case(V, B, 1, 4)
    temp = torch.full((B,), 0.8)
    fh = _filters(B, V, 2)
    fh.top_k = torch.tensor([-5, 0, 0, 0, 0, 0], dtype=torch.int32)
    fh.min_p = torch.tensor([0.0, float("nan"), 2.0, 0.0, 0.0, -1.0])
    fh.repetition_penalty = torch.tensor([1.0, 1.0, 1.0, -2.0, float("inf"), 1.0])
    fh.presence_penalty = torch.tensor([0.0, 0.0, 0.0, float("nan"), 0.0, 0.0])
    fh.frequency_penalty = torch.tensor([0.0, 0.0, 0.0, 0.0, float("-inf"), float("nan")])
    neutral = _to(_filters(B, V, 2, neutral=True))
    neutral.table.copy_(fh.table.to(DEV))
    neutral.min_p[2] = 1.0   # min_p > 1 is taken as 1
    outs = []
    for f in (_to(fh), neutral):
        dbg = torch.zeros((B, 8), dtype=torch.int64, device=DEV)
        dw = torch.zeros((B, V), device=DEV)
        tok = sample(logits[:, 0].to(DEV), temp.to(DEV), top.to(DEV), 9, torch.tensor([1], device=DEV), debug=dbg, debug_w=dw,
                     filters=f)
        outs.append((tok.cpu(), dbg.cpu(), dw.cpu()))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def _chi2(counts, probs):
    keep = probs > 0
    assert counts[~keep].sum() == 0
    return stats.chisquare(counts[keep], probs[keep] / probs[keep].sum() * counts[keep].sum()).pvalue


def _filtered_law(l, T, p, vals, table_row, drafts=()):
    l3 = F.penalised(l, table_row, F.draft_counts(drafts, len(l)), vals)
    W = R.fixed_point(R.weights_fp64(l3, T))
    keep, _ = F.truncate(W, p, vals)
    q = np.where(keep, W, 0).astype(np.float64)
    return q / q.sum()


def test_chi_square(cuda_lib):
    """200 000 draws: the first token follows the filtered law and not the unfiltered one; with a fixed draft d the second
    emitted token, given d accepted, follows the filtered law that counts d (exactness under drafts)."""
    V, Bq, n_off, Tt, p = 200, 2000, 100, 0.9, 0.95
    g = torch.Generator().manual_seed(5)
    rows = torch.randn((2, V), generator=g) * 1.5
    trow = np.zeros(V, dtype=np.int64)
    trow[:30] = 1 << 31
    trow[30:40] = 2
    vals = F.device_values(top_k=40, min_p=0.02, repetition_penalty=1.4, presence_penalty=0.3, frequency_penalty=0.2)
    q0 = _filtered_law(rows[0].numpy(), Tt, p, vals, trow)
    q1_ignoring = _filtered_law(rows[1].numpy(), Tt, p, vals, trow)
    d = int(np.argmax(q0 * q1_ignoring))   # kept in both rows, so counting d in row 1 changes its law
    q1 = _filtered_law(rows[1].numpy(), Tt, p, vals, trow, drafts=[d])
    fh = SampleFilters.neutral(Bq, V, "cpu")
    fh.top_k.fill_(40)
    fh.min_p.fill_(0.02)
    fh.repetition_penalty.fill_(1.4)
    fh.presence_penalty.fill_(0.3)
    fh.frequency_penalty.fill_(0.2)
    f = _to(fh)
    base = torch.from_numpy(trow.astype(np.uint32).view(np.int32)).to(DEV)
    logits = rows[None].expand(Bq, 2, V).contiguous().to(DEV)
    temp, top = torch.full((Bq,), Tt, device=DEV), torch.full((Bq,), p, device=DEV)
    ids = torch.zeros((Bq, 2), dtype=torch.int64, device=DEV)
    hist = torch.zeros((Bq, 2), dtype=torch.int32, device=DEV)
    length, limit, done = (torch.zeros(Bq, dtype=torch.int32, device=DEV), torch.full((Bq,), 2, dtype=torch.int32, device=DEV),
                           torch.zeros(Bq, dtype=torch.int32, device=DEV))
    offset = torch.zeros(1, dtype=torch.int64, device=DEV)
    first, second = np.zeros(V), np.zeros(V)
    for o in range(n_off):
        ids[:, 1] = d
        length.zero_()
        done.zero_()
        f.table.copy_(base.expand(Bq, V))
        offset.fill_(o)
        verify_sample(logits, temp, top, 99, offset, ids, history=hist, length=length, limit=limit, done=done, filters=f)
        h, n = hist.cpu().numpy(), length.cpu().numpy()
        first += np.bincount(h[:, 0], minlength=V)
        a = n == 2
        second += np.bincount(h[a, 1], minlength=V)
    assert _chi2(first, q0) > 1e-3
    assert _chi2(second, q1) > 1e-3
    unfiltered = _filtered_law(rows[0].numpy(), Tt, p, F.device_values(), trow)
    assert stats.chisquare(first[unfiltered > 0], unfiltered[unfiltered > 0] * first.sum()).pvalue < 1e-6
    # the law that ignores the draft is rejected: draws outside its support, or a chi-square p-value below 1e-6
    inside = q1_ignoring > 0
    assert not np.allclose(q1, q1_ignoring)
    assert second[~inside].sum() > 0 or stats.chisquare(second[inside], q1_ignoring[inside] * second.sum()).pvalue < 1e-6


def test_table_bookkeeping(cuda_lib):
    """sample() counts each token it appends to the record and nothing for a request already done or without a record; the
    verification call counts emitted tokens only (accepted drafts and the final token), nothing for a done request."""
    V, B = 1000, 3
    g = torch.Generator().manual_seed(2)
    logits = torch.randn((B, V), generator=g).to(DEV)
    fh = SampleFilters.neutral(B, V, "cpu")
    fh.repetition_penalty.fill_(1.1)
    f = _to(fh)
    temp, top, off = torch.zeros(B, device=DEV), torch.ones(B, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    toks = torch.zeros((B, 4), dtype=torch.int32, device=DEV)
    count = torch.zeros(B, dtype=torch.int32, device=DEV)
    done = torch.tensor([0, 1, 0], dtype=torch.int32, device=DEV)
    ids = sample(logits, temp, top, 1, off, tokens_out=toks, count=count, done=done, filters=f)
    tab = f.table.cpu()
    for b in range(B):
        want = np.zeros(V, dtype=np.int64)
        if b != 1:
            want[int(ids[b])] = 1
        assert tab[b].numpy().tolist() == want.tolist()
    sample(logits, temp, top, 1, off, filters=f)   # no record: nothing counted
    assert torch.equal(f.table.cpu(), tab)
    # verification: greedy drafts d1 = argmax (accepted), d2 = not the argmax (rejected)
    T = 3
    lg = torch.randn((B, T, V), generator=g).to(DEV)
    f.table.zero_()
    f.repetition_penalty.fill_(1.0)
    f.frequency_penalty.fill_(0.5)
    vid = torch.zeros((B, T), dtype=torch.int64, device=DEV)
    vid[:, 1] = lg[:, 0].argmax(-1)
    vid[:, 2] = (lg[:, 1].argmax(-1) + 1) % V
    hist = torch.zeros((B, 10), dtype=torch.int32, device=DEV)
    length, limit = torch.zeros(B, dtype=torch.int32, device=DEV), torch.full((B,), 10, dtype=torch.int32, device=DEV)
    done = torch.tensor([0, 1, 0], dtype=torch.int32, device=DEV)
    verify_sample(lg, temp, top, 1, off, vid, history=hist, length=length, limit=limit, done=done, filters=f)
    tab, h, n = f.table.cpu(), hist.cpu(), length.cpu()
    for b in range(B):
        want = np.zeros(V, dtype=np.int64)
        for x in h[b, :int(n[b])].tolist():
            want[x] += 1
        assert tab[b].numpy().tolist() == want.tolist()
    assert n.tolist() == [2, 0, 2]


def test_capture_picks_up_new_values(cuda_lib):
    """A captured filtered sample() reads the per-request values at replay time."""
    V, B = 32000, 8
    logits, temp, top, _ = _case(V, B, 1, 6)
    lg, tp, pp = logits[:, 0].to(DEV), torch.full((B,), 0.8, device=DEV), top.to(DEV)
    f = _to(_filters(B, V, 3))
    off = torch.zeros(1, dtype=torch.int64, device=DEV)
    ids = torch.zeros((B,), dtype=torch.int64, device=DEV)
    dbg = torch.zeros((B, 8), dtype=torch.int64, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sample(lg, tp, pp, 4, off, ids_out=ids, debug=dbg, filters=f)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sample(lg, tp, pp, 4, off, ids_out=ids, debug=dbg, filters=f)
    for k_top in (1, 7, 0):
        f.top_k.fill_(k_top)
        f.min_p.fill_(0.0)
        graph.replay()
        torch.cuda.synchronize()
        got = (ids.clone(), dbg.clone())
        e_ids, e_dbg = torch.zeros_like(ids), torch.zeros_like(dbg)
        sample(lg, tp, pp, 4, off, ids_out=e_ids, debug=e_dbg, filters=f)
        assert torch.equal(got[0], e_ids) and torch.equal(got[1], e_dbg)
        assert (got[1][:, 5] == (k_top if k_top else V)).all()


# ---- generate() with filters ------------------------------------------------------------------------------------------------------
GEN_BUF = 16
FILT = dict(top_k=[0, 20], min_p=0.05, repetition_penalty=1.3, presence_penalty=0.4, frequency_penalty=0.2)


def _runner(B=2):
    from magicpig_b200.llama_runner import LlamaDecodeRunner, LlamaShape
    shape = LlamaShape("tiny", 3, 512, 1024, 4, 2, 1000, 500000.0, 1e-5)
    return LlamaDecodeRunner(shape, 6, 16, B, 512, device=DEV, seed=3, generation_buffer=GEN_BUF, dense_layers=(0,), fused=False,
                             max_query_tokens=8)


def _ids(n, seed, period=0):
    x = torch.randint(0, 1000, (n,), generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)
    if period:
        x = x[:period].repeat(n // period + 1)[:n]
    return x


def _eager(run, prompts, n_new, temp, top_p, seed, k):
    """generate(..., **FILT, draft_tokens=k) by hand with the same calls, eagerly."""
    from magicpig_b200.llama_runner import spec_spill_every
    srv, B = run.server, run.B
    for b, pr in enumerate(prompts):
        run.prefill(pr, request=b)
    run.set_sampling(temp, top_p, seed=seed, offset=0, **FILT)
    ops.penalty_table(prompts, run.shape.vocab_size, out=run._penalty_table())
    if k == 0:
        tokens, count, done = run._gen_record()
        count.zero_()
        done.zero_()
        run.sample()
        used = 0
        for _ in range(n_new - 1):
            if used == run.generation_buffer:
                srv.spill_window()
                used = 0
            run.step()
            run.sample()
            used += 1
        n = count.tolist()
        return [tokens[b, :n[b]].tolist() for b in range(B)]
    hist, length, limit, done = run._history()
    P = [int(p.numel()) for p in prompts]
    for b in range(B):
        hist[b, :P[b]] = prompts[b].int()
    length.copy_(torch.tensor(P, dtype=torch.int32))
    limit.copy_(torch.tensor([x + n_new for x in P], dtype=torch.int32))
    done.zero_()
    run._verify(run.logits[:, None], count=False)
    run.sample_offset.add_(1)
    every, since = spec_spill_every(GEN_BUF, k), 0
    for _ in range(n_new - 1):
        if since == every:
            srv.spill_window()
            since = 0
        run.spec_step(k + 1)
        since += 1
    n = length.tolist()
    return [hist[b, P[b]:n[b]].tolist() for b in range(B)]


@pytest.mark.parametrize("k", [0, 1, 3])
@pytest.mark.parametrize("temp", [0.0, 0.7])
def test_generate_equals_eager_loop(cuda_lib, k, temp):
    prompts = [_ids(300, 1, period=37), _ids(257, 2, period=11)]
    run = _runner()
    out = run.generate(prompts, 40, temperature=temp, top_p=0.9, seed=9, check_every=4, draft_tokens=k, **FILT)
    ref = _eager(_runner(), prompts, 40, temp, 0.9, 9, k)
    assert out == ref and [len(o) for o in out] == [40, 40]
    # the table holds the prompt bits and the emitted tokens' counts
    tab = run.penalty_table.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    for b in range(2):
        want = np.zeros(1000, dtype=np.int64)
        want[prompts[b].cpu().numpy()] = 1 << 31
        for x in out[b]:
            want[x] += 1
        assert tab[b].tolist() == want.tolist()
    # neutral filters afterwards: the unfiltered graph, the same tokens as a runner that never saw filters
    plain = run.generate(prompts, 20, temperature=temp, top_p=0.9, seed=9, draft_tokens=k)
    assert plain == _runner().generate(prompts, 20, temperature=temp, top_p=0.9, seed=9, draft_tokens=k)


def test_generate_refuses_bad_filters(cuda_lib):
    run = _runner()
    for kw in (dict(min_p=1.5), dict(repetition_penalty=0.0), dict(presence_penalty=3.0), dict(top_k=[1, 2, 3])):
        with pytest.raises(ValueError):
            run.generate(_ids(300, 1), 10, **kw)
    assert run._gen_graph is None and run.penalty_table is None and run.pos.tolist() == [0, 0]
