"""Speculative decoding without a GPU: the restatement of mpig_aux_verify_sample's rule in tests/support/spec_rule.py is lossless in
exact rational arithmetic and tells the named mistakes apart; the restatement of mpig_aux_ngram_draft's rule on hand-made
histories; the ctypes bindings against the aux header; the wrappers' and generate()'s refusals; the spill cadence."""
import ctypes
import math
import re
from fractions import Fraction

import numpy as np
import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200.llama_runner import check_spec_args, spec_spill_every
from magicpig_b200.ops import MAX_NGRAM, MAX_VERIFY_TOKENS, check_ngram_args, check_verify_args
from tests.support import sample_rule as R
from tests.support import spec_rule as S

# small integer weights: a nucleus boundary inside a tie (p = 0.6 of S = 11 -> floor 6: tokens 0..2 kept, token 3 ties tokens 1, 2
# and falls outside), an outside token and a zero weight.  The kept and residual masses 8, 6, 4 keep the exact enumeration small.
W_SMALL = [4, 2, 2, 2, 1, 0]
P_SMALL = 0.6


def _word(i, M):
    """A 64-bit word whose umulhi64 with any S dividing M is floor(i S / M): uniform i in [0, M) makes every such target uniform."""
    return -(-(i << 64) // M)


def _first_token_law(W, p, d, mistake=None):
    """P(first emitted token = x) over independent uniform acceptance and residual words, exactly (Fraction)."""
    W = np.asarray(W, dtype=np.int64)
    keep = R.keep_mask(W, R.nucleus_threshold(p, int(W.sum())))
    S_keep = int(np.where(keep, W, 0).sum())
    masses = {S_keep} | {S_keep - int(W[x]) for x in range(len(W)) if keep[x] and S_keep - int(W[x]) > 0}
    M = math.lcm(*masses)
    law = {}
    for ia in range(M):
        ra = _word(ia, M)
        for i0 in range(M):
            acc, final, _ = S.row_from_weights(W, p, _word(i0, M), ra, d, mistake)
            x = d if acc else final
            law[x] = law.get(x, 0) + 1
    return {x: Fraction(c, M * M) for x, c in law.items()}, keep, S_keep


def _nucleus_law(W, keep, S_keep):
    return {x: Fraction(int(W[x]), S_keep) for x in range(len(W)) if keep[x] and W[x] > 0}


# ---- the acceptance rule is lossless ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", list(range(len(W_SMALL))) + [None, 99])
def test_first_token_follows_the_nucleus(d):
    """For every draft (the argmax, a kept token, the kept and the dropped side of a boundary tie, a token outside the nucleus, a
    zero weight, none, an id outside the vocabulary) the first emitted token has probability W_x / S_keep."""
    law, keep, S_keep = _first_token_law(W_SMALL, P_SMALL, d)
    assert keep.tolist() == [True, True, True, False, False, False]   # the tie at 2 is split
    assert law == _nucleus_law(np.asarray(W_SMALL), keep, S_keep)


def test_acceptance_rate_is_p_of_d():
    W = np.asarray(W_SMALL)
    keep = R.keep_mask(W, R.nucleus_threshold(P_SMALL, int(W.sum())))
    S_keep = int(np.where(keep, W, 0).sum())
    M = S_keep
    for d in range(len(W)):
        n = sum(S.row_from_weights(W, P_SMALL, 0, _word(i, M), d)[0] for i in range(M))
        assert Fraction(n, M) == (Fraction(int(W[d]), S_keep) if keep[d] else 0)


@pytest.mark.parametrize("mistake", ["no_exclude", "reuse_word", "le"])
def test_named_row_mistakes_change_the_law(mistake):
    """Each wrong row rule moves the first token's law away from the nucleus for some draft."""
    W = np.asarray(W_SMALL)
    moved = False
    for d in range(len(W)):
        law, keep, S_keep = _first_token_law(W, P_SMALL, d, mistake)
        moved |= law != _nucleus_law(W, keep, S_keep)
    assert moved


def test_drop_off_by_one_and_next_row_are_told_apart():
    rows = [(True, 5, False), (False, 7, False), (False, 9, False), (True, 11, False)]
    good = S.resolve(rows, [3, 4, 6])
    assert good["k"] == 1 and good["final"] == 7 and good["drop"] == 2 and good["emitted"] == [3, 7]
    assert S.resolve(rows, [3, 4, 6], mistake="drop_off")["drop"] != good["drop"]
    assert S.resolve(rows, [3, 4, 6], mistake="next_row")["final"] != good["final"]


def test_bookkeeping():
    rows = [(True, 5, False), (True, 7, False), (False, 9, False)]
    r = S.resolve(rows, [3, 4], eos=(3,))
    assert r["emitted"] == [3] and r["done"] and r["drop"] == 2                 # EOS among the drafts: kept, then stop
    r = S.resolve(rows, [3, 4], length=10, limit=12)
    assert r["emitted"] == [3, 4] and r["done"] and r["drop"] == 1              # the limit: only the emitted tokens' rows stay
    r = S.resolve(rows, [3, 4], length=10, limit=13)
    assert r["emitted"] == [3, 4, 9] and r["done"] and r["drop"] == 0           # the limit on the final token
    r = S.resolve(rows, [3, 4], done=True)
    assert r["emitted"] == [] and r["drop"] == 3 and not r["counted"]           # a done request rewinds its whole step
    r = S.resolve([(True, 5, False), (False, 0, True), (False, 9, False)], [3, 4])
    assert r["k"] == 1 and r["final"] == 0 and r["invalid"]                     # an invalid row ends acceptance


def test_t1_is_sample():
    rng = np.random.default_rng(3)
    for i in range(50):
        logits = rng.normal(size=300).astype(np.float32) * 3
        out = S.request([logits], 0.6, 0.9, 77, 5 + i, 2, [0])
        assert out["final"] == R.sample_row(logits, 0.6, 0.9, 77, 5 + i, 2)[0]
        assert out["rows"][0][3][:5] == R.sample_row(logits, 0.6, 0.9, 77, 5 + i, 2)[1]


def test_greedy_rows():
    logits = np.array([[0, 3, 3, 1], [5, 0, 0, 0], [0, 0, 0, 9]], dtype=np.float32)
    out = S.request(logits, 0.0, 0.9, 1, 0, 0, [0, 1, 1])
    assert out["k"] == 1 and out["final"] == 0 and out["emitted"] == [1, 0]


# ---- prompt lookup --------------------------------------------------------------------------------------------------------------
def test_ngram_longest_then_most_recent():
    h = [1, 2, 3, 9, 2, 3, 8, 5, 3, 7, 2, 3]
    # suffix (2, 3): ends 2 and 5 match 2 tokens (h[1..2], h[4..5]); end 8 matches 1; the most recent 2-match is 5
    assert S.ngram_choice(h) == 5
    assert S.ngram_drafts(h, 4) == [8, 5, 3]


def test_ngram_overlapping_copy():
    h = [4, 1, 2, 1, 2, 1, 2]
    assert S.ngram_choice(h) == 4   # (1, 2) ending at 4 matches 3 tokens; ending at 6 is the suffix itself, outside [0, n - 2]
    assert S.ngram_drafts(h, 8) == [1, 2, 1, 2, 1, 2, 1]   # runs past the history into the drafts


def test_ngram_no_match_and_g_min():
    assert S.ngram_drafts([1, 2, 3, 4], 3) == [4, 4]
    assert S.ngram_drafts([7], 3) == [7, 7]
    assert S.ngram_drafts([], 3) == [0, 0]
    h = [5, 6, 1, 7, 6]
    assert S.ngram_choice(h, 1) == 1
    assert S.ngram_choice(h, 2) is None and S.ngram_drafts(h, 3, g_min=2) == [6, 6]


def test_ngram_match_ending_at_n_minus_2():
    assert S.ngram_choice([3, 8, 8]) == 1 and S.ngram_drafts([3, 8, 8], 4) == [8, 8, 8]


def test_ngram_g_max_caps_the_match():
    h = [1, 2, 3, 4, 0, 1, 2, 3, 4, 9, 2, 3, 4]
    assert S.ngram_choice(h, 1, 3) == 8 and S.ngram_choice(h, 1, 4) == 8
    assert S.ngram_choice(h, 1, 2) == 8
    h2 = [1, 2, 3, 4, 0, 9, 3, 4, 5, 1, 2, 3, 4]
    assert S.ngram_choice(h2, 1, 2) == 7 and S.ngram_choice(h2, 1, 4) == 3


# ---- the C ABI and the wrappers -------------------------------------------------------------------------------------------------
def _aux_prototype(name):
    text = re.sub(r"/\*.*?\*/", "", open(N.AUX_HEADER_PATH).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)", text)
    assert m, f"{name} not declared"
    return [p.strip() for p in m.group(1).split(",")]


def _ctypes_of(params):
    want = []
    for p in params:
        if "*" in p:
            want.append(ctypes.c_void_p)
        elif p.startswith("int64_t"):
            want.append(ctypes.c_int64)
        elif p.startswith("uint64_t"):
            want.append(ctypes.c_uint64)
        else:
            assert re.match(r"int\s+\w+$", p), p
            want.append(ctypes.c_int)
    return want


@pytest.mark.parametrize("name,names", [
    ("mpig_aux_verify_sample", ["logits", "B", "T", "V", "ld_b", "ld_t", "temperature", "top_p", "seed", "offset", "ids", "ids_stride",
                                "rows", "drop", "history", "history_ld", "length", "limit", "done", "steps", "accepted", "eos_ids",
                                "n_eos", "status", "debug", "debug_w", "stream"]),
    ("mpig_aux_ngram_draft", ["history", "B", "ld", "length", "ids", "ids_stride", "T", "g_min", "g_max", "stream"]),
])
def test_binding_matches_header(name, names):
    params = _aux_prototype(name)
    res, args = N._AUX_SIGNATURES[name]
    assert res is ctypes.c_int and args == _ctypes_of(params)
    assert [re.sub(r".*\W", "", p) for p in params] == names
    assert name in N.declared_symbols(N.AUX_HEADER_PATH)


def _vargs(B=3, T=4, V=100):
    i32 = lambda *s: torch.zeros(s, dtype=torch.int32)  # noqa: E731
    return dict(logits=torch.zeros((B, 8, V))[:, :T], temperature=torch.ones(B), top_p=torch.ones(B),
                offset=torch.zeros(1, dtype=torch.int64), ids=torch.zeros((B, 8), dtype=torch.int64), drop=i32(B),
                history=i32(B, 50), length=i32(B), limit=i32(B), done=i32(B), steps=i32(B), accepted=i32(B),
                status=i32(1), debug=torch.zeros((B, T, 9), dtype=torch.int64), debug_w=torch.zeros((B, T, V)))


def test_verify_wrapper_accepts():
    rows, eos = check_verify_args(**_vargs(), eos_token_ids=range(8))
    assert rows.shape == (3, 4, 2) and rows.dtype == torch.int32 and eos == list(range(8))
    a = _vargs(T=1)
    a["logits"] = torch.zeros((3, 100))[:, None]   # the (B, V) logits of a single-token step
    check_verify_args(**a)


@pytest.mark.parametrize("what", ["rank", "T0", "T9", "dtype", "cols_strided", "rows_overlap", "temperature", "ids_dtype", "ids_short",
                                  "ids_strided", "rows_shape", "history_alone", "limit_missing", "steps_alone", "drop_dtype",
                                  "debug_shape", "debug_w_shape", "eos_count"])
def test_verify_wrapper_refusals(what):
    a = _vargs()
    if what == "rank":
        a["logits"] = torch.zeros((3, 100))
    elif what == "T0":
        a["logits"] = torch.zeros((3, 0, 100))
    elif what == "T9":
        a["logits"] = torch.zeros((3, MAX_VERIFY_TOKENS + 1, 100))
    elif what == "dtype":
        a["logits"] = a["logits"].double()
    elif what == "cols_strided":
        a["logits"] = torch.zeros((3, 4, 200))[:, :, ::2]
    elif what == "rows_overlap":
        a["logits"] = torch.zeros(1000).as_strided((3, 4, 100), (100, 50, 1))
    elif what == "temperature":
        a["temperature"] = torch.ones(2)
    elif what == "ids_dtype":
        a["ids"] = a["ids"].int()
    elif what == "ids_short":
        a["ids"] = torch.zeros((3, 3), dtype=torch.int64)
    elif what == "ids_strided":
        a["ids"] = torch.zeros((3, 16), dtype=torch.int64)[:, ::2]
    elif what == "rows_shape":
        a["rows"] = torch.zeros((3, 4), dtype=torch.int32)
    elif what == "history_alone":
        del a["length"], a["limit"], a["done"]
    elif what == "limit_missing":
        del a["limit"]
    elif what == "steps_alone":
        del a["accepted"]
    elif what == "drop_dtype":
        a["drop"] = torch.zeros(3, dtype=torch.int64)
    elif what == "debug_shape":
        a["debug"] = torch.zeros((3, 4, 5), dtype=torch.int64)
    elif what == "debug_w_shape":
        a["debug_w"] = torch.zeros((3, 100))
    elif what == "eos_count":
        a["eos_token_ids"] = range(9)
    with pytest.raises(N.MagicPigError):
        check_verify_args(**a)


def _nargs(B=2):
    return dict(history=torch.zeros((B, 64), dtype=torch.int32), length=torch.zeros(B, dtype=torch.int32),
                ids=torch.zeros((B, 8), dtype=torch.int64), T=4, g_min=1, g_max=3)


def test_ngram_wrapper_accepts():
    check_ngram_args(**_nargs())
    check_ngram_args(**dict(_nargs(), T=1, g_min=MAX_NGRAM, g_max=MAX_NGRAM))


@pytest.mark.parametrize("kw", [dict(T=0), dict(T=9), dict(g_min=0), dict(g_max=9), dict(g_min=3, g_max=2),
                                dict(history=torch.zeros((2, 64), dtype=torch.int64)), dict(history=torch.zeros(64, dtype=torch.int32)),
                                dict(history=torch.zeros((2, 128), dtype=torch.int32)[:, ::2]),
                                dict(length=torch.zeros(3, dtype=torch.int32)), dict(length=torch.zeros(2, dtype=torch.int64)),
                                dict(ids=torch.zeros((2, 3), dtype=torch.int64)), dict(ids=torch.zeros((3, 8), dtype=torch.int64)),
                                dict(ids=torch.zeros((2, 8), dtype=torch.int32))])
def test_ngram_wrapper_refusals(kw):
    with pytest.raises(N.MagicPigError):
        check_ngram_args(**dict(_nargs(), **kw))


# ---- generate(draft_tokens=k) ---------------------------------------------------------------------------------------------------
def _spec_args(**kw):
    a = dict(lengths=[300], max_new_tokens=40, draft_tokens=3, ngram=(1, 3), max_query_tokens=8, generation_buffer=16, max_length=512,
             dense_tail_rows=0, can_spill=True)
    a.update(kw)
    return a


def test_spec_args_accepted():
    check_spec_args(**_spec_args())
    check_spec_args(**_spec_args(lengths=[300, 469]))                 # 469 + 40 + 3 = max_length
    check_spec_args(**_spec_args(draft_tokens=7, generation_buffer=8))
    check_spec_args(**_spec_args(dense_tail_rows=43))                 # 40 + 3 rows after the prompt at most
    check_spec_args(**_spec_args(can_spill=False, max_new_tokens=5))  # 4 replays of 4 rows fit the 16-row window
    check_spec_args(**_spec_args(ngram=(8, 8)))


@pytest.mark.parametrize("kw", [dict(draft_tokens=-1), dict(draft_tokens=8), dict(max_query_tokens=3), dict(generation_buffer=3),
                                dict(lengths=[300, 470]), dict(dense_tail_rows=42), dict(ngram=(0, 3)), dict(ngram=(1, 9)),
                                dict(can_spill=False, max_new_tokens=6), dict(can_spill=False, draft_tokens=1, max_new_tokens=10),
                                dict(ngram=(3, 2))])
def test_spec_args_refused(kw):
    with pytest.raises(ValueError):
        check_spec_args(**_spec_args(**kw))


@pytest.mark.parametrize("gb,k", [(256, 1), (256, 3), (256, 7), (16, 3), (8, 7), (5, 4)])
def test_spill_cadence(gb, k):
    """Replays between spills: every replay holds k + 1 rows during its step and keeps at most k + 1, so `every` replays never need
    more than the window and one more would overflow it when every draft is accepted."""
    every = spec_spill_every(gb, k)
    assert every >= 1 and every * (k + 1) <= gb < (every + 1) * (k + 1)
