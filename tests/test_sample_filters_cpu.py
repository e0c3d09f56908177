"""Sampling filters without a GPU: the restatement in tests/support/filter_rule.py equals a Hugging Face-style torch processor chain,
tells the named mistakes apart and is lossless under drafts in exact rational arithmetic; the ctypes bindings and struct against
the aux header; the ops and generate() refusals; penalty_table."""
import ctypes
import re
from fractions import Fraction

import numpy as np
import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200 import ops
from magicpig_b200.llama_runner import check_generate_args, filter_values
from tests.support import filter_rule as F
from tests.support import sample_rule as R


# ---- the restatement against a Hugging Face-style chain ------------------------------------------------------------------------
def _hf_keep(logits, table_row, T, top_k, top_p, min_p, r, pr, f):
    """Hugging Face's processors in its order on fp64: repetition (prompt + output), presence / frequency (output), temperature,
    top-k mask, top-p over the renormalised remainder, min-p relative to the max.  Returns the kept mask."""
    l = torch.tensor(logits, dtype=torch.float64)
    e = torch.tensor(table_row.astype(np.int64))
    c = (e & F.COUNT_MASK).double()
    seen = ((e >> 31) & 1).bool() | (c > 0)
    l = torch.where(seen, torch.where(l > 0, l / r, l * r), l)
    l = l - f * c - pr * (c > 0).double()
    p = torch.softmax(l / T, 0)
    order = torch.argsort(-p, stable=True)
    keep = torch.zeros_like(p, dtype=torch.bool)
    kset = order[:top_k] if top_k > 0 else order
    q = torch.zeros_like(p)
    q[kset] = p[kset]
    q = q / q.sum()
    cum = torch.cumsum(q[order], 0)
    keep_p = torch.zeros_like(keep)
    keep_p[order] = (cum - q[order]) <= top_p
    keep[kset] = True
    keep &= keep_p
    keep &= p >= min_p * p.max()
    return keep.numpy()


@pytest.mark.parametrize("seed", range(12))
def test_keep_set_equals_hf_chain(seed):
    g = np.random.default_rng(seed)
    V = 64
    logits = g.normal(0, 2, V).astype(np.float32)
    table = np.zeros(V, dtype=np.uint64)
    table[g.choice(V, 8, replace=False)] |= F.PROMPT_BIT
    table[g.choice(V, 6, replace=False)] += g.integers(1, 4, 6).astype(np.uint64)
    T = float(np.float32(g.choice([0.6, 1.0, 1.3])))
    top_k, top_p, min_p = int(g.choice([0, 5, 20])), float(np.float32(g.choice([0.8, 0.95, 1.0]))), float(np.float32(g.choice([0.0, 0.05])))
    vals = F.device_values(top_k, min_p, 1.3, 0.4, 0.3)
    l3 = F.penalised(logits, table, None, vals)
    W = R.fixed_point(R.weights_fp64(l3, T))
    keep, _ = F.truncate(W, top_p, vals)
    want = _hf_keep(logits, table, T, top_k, top_p, min_p, float(vals["r"]), float(vals["pr"]), float(vals["f"]))
    assert keep.tolist() == want.tolist()


# ---- the named mistakes ----------------------------------------------------------------------------------------------------------
def _case(mistake):
    """A row where `mistake` changes the kept set or the penalised logits."""
    V = 12
    logits = np.array([5.0, 3.0, 2.5, 2.5, 2.0, 1.0, 0.5, -1.0, 4.0, 2.5, -2.0, 0.0], dtype=np.float32)
    table = np.zeros(V, dtype=np.uint64)
    table[[0, 7]] |= F.PROMPT_BIT
    table[[8, 5]] += np.array([2, 1], dtype=np.uint64)
    kw = dict(top_k=4, min_p=0.1, repetition_penalty=1.5, presence_penalty=0.5, frequency_penalty=0.4)
    return logits, table, kw


@pytest.mark.parametrize("mistake", ["p_from_S", "minp_first", "minp_sum", "pos_times_r", "freq_after_temp", "prompt_counted",
                                     "topk_ties_high"])
def test_named_mistakes_change_the_result(mistake):
    logits, table, kw = _case(mistake)
    T, p = 0.7, 0.6
    if mistake == "topk_ties_high":   # the top-k boundary inside the tie at 2.5 (tokens 2, 3, 9)
        kw.update(top_k=4, min_p=0.0, repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0)
        p = 1.0
    if mistake == "minp_first":
        kw.update(top_k=0, min_p=0.3)
        p = 0.7
    if mistake == "minp_sum":
        kw.update(top_k=0, min_p=0.3)
        p = 1.0
    if mistake == "p_from_S":
        kw.update(min_p=0.0)
    vals = F.device_values(**kw)

    def result(m):
        l3 = F.penalised(logits, table, None, vals, T, m)
        W = R.fixed_point(R.weights_fp64(l3, T))
        keep, info = F.truncate(W, p, vals, m)
        return keep.tolist(), W.tolist()
    assert result(mistake) != result(None), mistake


def test_ignoring_drafts_changes_the_verification_row():
    logits, table, kw = _case(None)
    vals = F.device_values(**kw)
    rows = [F.verify_row(logits, 0.7, 0.9, vals, table, [8, 8], 3, 5, 0, 2, 1, mistake=m)[3] for m in (None, "ignore_drafts")]
    assert rows[0] != rows[1]


# ---- lossless under drafts, exactly ---------------------------------------------------------------------------------------------
def _small_weights(l3):
    """A weight map onto small integers (W = max(l3, 0) of integer-valued logits) that keeps the exact enumeration small; the
    acceptance, the residual and the truncation are the contract's, on these weights."""
    return np.maximum(np.asarray(l3, dtype=np.float64), 0).astype(np.int64)


def _row_law(W, keep, d, am):
    """P(the row emits x first) over uniform acceptance and residual words, exactly: the acceptance word over S_keep equally
    likely targets, the residual word over S_res (spec_rule's _word construction, one word at a time: they are independent)."""
    kept_w = np.where(keep, W, 0)
    S_keep = int(kept_w.sum())
    word = lambda i, M: -(-(i << 64) // M)  # noqa: E731
    law = {}
    acc = sum(F.row_from_keep(W, keep, 0, word(i, S_keep), d, am)[0] for i in range(S_keep))
    if acc:
        law[d] = Fraction(acc, S_keep)
    S_res = F.row_from_keep(W, keep, 0, 0, d, am)[2][4]
    for i in range(max(S_res, 1)):
        acc_never = F.row_from_keep(W, keep, word(i, max(S_res, 1)), (1 << 64) - 1, d, am)
        x = acc_never[1]
        law[x] = law.get(x, 0) + Fraction(S_keep - acc, S_keep) / max(S_res, 1)
    return law


@pytest.mark.parametrize("T", [2, 3, 4])
@pytest.mark.parametrize("drafts", [(0, 0, 0), (1, 3, 1), (0, 2, 5)])
def test_each_position_follows_the_filtered_law_given_its_prefix(T, drafts):
    """Row t with its drafts d_1 .. d_t counted emits its token with the law that non-speculative sampling uses after emitting
    d_1 .. d_t (the table with those counts), for every row of the step; ignoring the drafts breaks it."""
    V = 6
    base = np.array([7, 6, 5, 5, 3, 2], dtype=np.float32)
    table = np.zeros(V, dtype=np.uint64)
    table[4] |= F.PROMPT_BIT
    table[1] += 1
    vals = F.device_values(top_k=4, presence_penalty=1.0, frequency_penalty=1.0)
    p = 0.75
    for t in range(T):
        prefix = list(drafts[:t])
        d = drafts[t] if t < T - 1 else None
        # the speculative row
        l3 = F.penalised(base, table, F.draft_counts(prefix, V), vals)
        W = _small_weights(l3)
        keep, _ = F.truncate(W, p, vals)
        law = _row_law(W, keep, d, int(np.argmax(l3)))
        # non-speculative sampling after d_1 .. d_t were emitted: the table counts them
        tab = table.copy()
        for x in prefix:
            tab[x] += 1
        Wn = _small_weights(F.penalised(base, tab, None, vals))
        keep_n, _ = F.truncate(Wn, p, vals)
        S_keep = int(np.where(keep_n, Wn, 0).sum())
        want = {x: Fraction(int(Wn[x]), S_keep) for x in range(V) if keep_n[x] and Wn[x] > 0}
        assert {x: q for x, q in law.items() if q} == want, (t, law, want)
        if prefix:   # a row that ignores its drafts samples from the wrong law
            Wi = _small_weights(F.penalised(base, table, None, vals))
            assert Wi.tolist() != Wn.tolist()


# ---- the C ABI and the wrappers ---------------------------------------------------------------------------------------------------
def _aux_prototype(name):
    text = re.sub(r"/\*.*?\*/", "", open(N.AUX_HEADER_PATH).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)", text)
    assert m, f"{name} not declared"
    return [p.strip() for p in m.group(1).split(",")]


@pytest.mark.parametrize("name,base", [("mpig_aux_sample_filtered", "mpig_aux_sample"),
                                       ("mpig_aux_verify_sample_filtered", "mpig_aux_verify_sample")])
def test_binding_matches_header(name, base):
    params, base_params = _aux_prototype(name), _aux_prototype(base)
    assert params[:-2] == base_params[:-1] and params[-2:] == ["const mpig_sample_filters *filters", "void *stream"]
    res, args = N._AUX_SIGNATURES[name]
    assert res is ctypes.c_int and args[:-2] == N._AUX_SIGNATURES[base][1][:-1]
    assert args[-2] == ctypes.POINTER(N.MpigSampleFilters) and args[-1] is ctypes.c_void_p
    assert name in N.declared_symbols(N.AUX_HEADER_PATH)


def test_struct_layout_matches_header():
    text = open(N.AUX_HEADER_PATH).read()
    body = re.search(r"typedef struct mpig_sample_filters \{(.*?)\} mpig_sample_filters;", text, re.S).group(1)
    names = re.findall(r"(\w+);", body)
    assert names == [f[0] for f in N.MpigSampleFilters._fields_]
    assert ctypes.sizeof(N.MpigSampleFilters) == 7 * 8
    assert [getattr(N.MpigSampleFilters, n).offset for n in names] == [8 * i for i in range(7)]


def _filters(B=3, V=100, **over):
    f = ops.SampleFilters.neutral(B, V, "cpu")
    for k, v in over.items():
        setattr(f, k, v)
    return f


def test_filters_accepted():
    ops.check_filters(_filters(), 3, 100, torch.device("cpu"))
    f = _filters(top_k=torch.tensor([-1, 0, 50], dtype=torch.int32), min_p=torch.tensor([0.0, 0.5, 1.0]),
                 repetition_penalty=torch.tensor([0.5, 1.0, 2.0]), presence_penalty=torch.tensor([-2.0, 0.0, 2.0]),
                 frequency_penalty=torch.tensor([2.0, -2.0, 0.1]), table=torch.zeros((3, 128), dtype=torch.uint32))
    ops.check_filters(f, 3, 100, torch.device("cpu"))


@pytest.mark.parametrize("what", ["type", "top_k_dtype", "top_k_shape", "min_p_dtype", "table_dtype", "table_short", "table_rows",
                                  "table_strided", "min_p_range", "min_p_nan", "rep_zero", "rep_inf", "pres_range", "freq_range",
                                  "freq_nan"])
def test_filters_refused(what):
    B, V = 3, 100
    f = _filters()
    bad = {"top_k_dtype": ("top_k", torch.zeros(B, dtype=torch.int64)), "top_k_shape": ("top_k", torch.zeros(B + 1, dtype=torch.int32)),
           "min_p_dtype": ("min_p", torch.zeros(B, dtype=torch.float64)), "table_dtype": ("table", torch.zeros((B, V))),
           "table_short": ("table", torch.zeros((B, V - 1), dtype=torch.int32)),
           "table_rows": ("table", torch.zeros((B + 1, V), dtype=torch.int32)),
           "table_strided": ("table", torch.zeros((B, 2 * V), dtype=torch.int32)[:, ::2]),
           "min_p_range": ("min_p", torch.tensor([0.0, 1.5, 0.0])), "min_p_nan": ("min_p", torch.tensor([float("nan"), 0.0, 0.0])),
           "rep_zero": ("repetition_penalty", torch.tensor([1.0, 0.0, 1.0])),
           "rep_inf": ("repetition_penalty", torch.tensor([1.0, float("inf"), 1.0])),
           "pres_range": ("presence_penalty", torch.tensor([0.0, 0.0, -2.5])),
           "freq_range": ("frequency_penalty", torch.tensor([3.0, 0.0, 0.0])),
           "freq_nan": ("frequency_penalty", torch.tensor([0.0, float("nan"), 0.0]))}
    if what == "type":
        f = dict(top_k=None)
    else:
        setattr(f, *bad[what])
    with pytest.raises(N.MagicPigError):
        ops.check_filters(f, B, V, torch.device("cpu"))


def test_sample_and_verify_take_filters_keyword_only():
    import inspect
    for fn in (ops.sample, ops.verify_sample):
        prm = inspect.signature(fn).parameters["filters"]
        assert prm.kind is inspect.Parameter.KEYWORD_ONLY and prm.default is None
    B, V = 2, 50
    logits, t, p, off = torch.zeros((B, V)), torch.ones(B), torch.ones(B), torch.zeros(1, dtype=torch.int64)
    with pytest.raises(N.MagicPigError):   # checked before the device check: a (B, 5) debug with filters is refused
        ops.sample(logits, t, p, 0, off, debug=torch.zeros((B, 5), dtype=torch.int64), filters=_filters(B, V))
    with pytest.raises(N.MagicPigError):
        ops.sample(logits, t, p, 0, off, filters=_filters(B, V, min_p=torch.tensor([2.0, 0.0])))
    with pytest.raises(N.MagicPigError, match="CUDA"):   # valid arguments reach the device check
        ops.sample(logits, t, p, 0, off, debug=torch.zeros((B, 8), dtype=torch.int64), filters=_filters(B, V))
    with pytest.raises(N.MagicPigError, match="CUDA"):
        ops.verify_sample(torch.zeros((B, 2, V)), t, p, 0, off, torch.zeros((B, 2), dtype=torch.int64),
                          debug=torch.zeros((B, 2, 12), dtype=torch.int64), filters=_filters(B, V))
    with pytest.raises(N.MagicPigError):
        ops.verify_sample(torch.zeros((B, 2, V)), t, p, 0, off, torch.zeros((B, 2), dtype=torch.int64),
                          debug=torch.zeros((B, 2, 9), dtype=torch.int64), filters=_filters(B, V))


def test_penalty_table():
    out = torch.full((3, 12), 7, dtype=torch.int32)
    t = ops.penalty_table([torch.tensor([1, 4, 4, 9]), [], torch.tensor([0, 9])], 10, out=out)
    assert t is out
    u = out.view(torch.int32).numpy().astype(np.int64) & 0xFFFFFFFF
    want = np.zeros((3, 12), dtype=np.int64)
    want[0, [1, 4, 9]] = want[2, [0, 9]] = 1 << 31
    assert (u == want).all()
    t2 = ops.penalty_table(torch.tensor([[3, 3], [0, 1]]), 5)
    assert t2.dtype == torch.int32 and t2.shape == (2, 5) and (t2 != 0).sum() == 3
    tu = ops.penalty_table([[2]], 4, out=torch.zeros((1, 4), dtype=torch.uint32))
    assert int(tu.view(torch.int32)[0, 2]) == ops.PROMPT_BIT
    for args in (([[10]], 10), ([[-1]], 10), ([[1.5]], 10), ([[1], [2]], 10, torch.zeros((1, 10), dtype=torch.int32)),
                 ([[1]], 10, torch.zeros((1, 9), dtype=torch.int32)), ([[1]], 10, torch.zeros((1, 10), dtype=torch.int64))):
        with pytest.raises(N.MagicPigError):
            ops.penalty_table(*args[:2], out=args[2] if len(args) > 2 else None)


def _gen_args(**kw):
    a = dict(lengths=[300], max_new_tokens=20, check_every=16, eos=(), max_length=512, num_sink=4, num_local=64, chunk_size=8192,
             generation_buffer=16, can_spill=True, B=2)
    a.update(kw)
    return a


def test_generate_filter_args():
    check_generate_args(**_gen_args(filters=dict(top_k=[0, 40], min_p=0.05, repetition_penalty=1.2, presence_penalty=-2.0,
                                                 frequency_penalty=2.0)))
    check_generate_args(**_gen_args(filters=dict(F.NEUTRAL)))
    assert filter_values(2, top_k=3, min_p=None) == dict(top_k=[3, 3])


@pytest.mark.parametrize("kw", [dict(top_k=1.5), dict(top_k=[1, 2, 3]), dict(min_p=-0.1), dict(min_p=1.01), dict(min_p=float("nan")),
                                dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(repetition_penalty=float("inf")),
                                dict(presence_penalty=2.5), dict(frequency_penalty=-2.01), dict(frequency_penalty=float("nan"))])
def test_generate_filter_refusals(kw):
    f = dict(F.NEUTRAL)
    f.update(kw)
    with pytest.raises(ValueError):
        check_generate_args(**_gen_args(filters=f))
