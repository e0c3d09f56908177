"""Sampling without a GPU: the restatement of mpig_aux_sample's contract in tests/support/sample_rule.py (Philox4x32-10 against its
published known answers, the exact nucleus threshold, the keep set against the reference's top-p mask, the tie rule), the named
mistakes it rejects, the ctypes binding against the aux header, the wrapper's argument refusals and generate()'s argument checks."""
import ctypes
import math
import re
from fractions import Fraction

import numpy as np
import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200.llama_runner import (LLAMA31_70B, LLAMA31_8B, LlamaShape, check_generate_args, generate_prompts, per_request)
from magicpig_b200.ops import MAX_EOS_IDS, check_sample_args
from tests.support import sample_rule as R


# ---- Philox4x32-10 --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
    ((7, 1, 3, 0), (12345, 678), (0x2B5A1C29, 0x4C604927, 0x3F53FC0C, 0x7BC902B5)),
])
def test_philox_known_answers(ctr, key, want):
    """The Random123 known-answer vectors of Philox4x32-10, and one word of curand_Philox4x32_10 at a counter of the sampler's
    form (offset lo, offset hi, row, 0)."""
    assert R.philox4x32_10(ctr, key) == want


def test_draw_word_layout():
    x, y, _, _ = R.philox4x32_10((7, 1, 3, 0), (12345, 678))
    assert R.draw_word(12345 | 678 << 32, 7 | 1 << 32, 3) == x | y << 32


# ---- the nucleus threshold ------------------------------------------------------------------------------------------------------
def test_threshold_is_exact():
    rng = np.random.default_rng(0)
    for _ in range(2000):
        p = float(np.float32(rng.random()))
        S = int(rng.integers(1 << 40, 128256 << 40))
        assert R.nucleus_threshold(p, S) == math.floor(Fraction(p) * S)
    S = 5 << 40
    assert R.nucleus_threshold(1.0, S) == S and R.nucleus_threshold(2.0, S) == S
    assert R.nucleus_threshold(0.0, S) == 0 and R.nucleus_threshold(-1.0, S) == 0 and R.nucleus_threshold(float("nan"), S) == 0
    assert R.nucleus_threshold(float(np.float32(1e-40)), S) == math.floor(Fraction(float(np.float32(1e-40))) * S)   # subnormal p


# ---- the keep set against the reference's mask ----------------------------------------------------------------------------------
def reference_mask(probs: torch.Tensor, p: float) -> torch.Tensor:
    """The reference's top-p rule (models/utils.py, topp_temperature_decode), restated: sort descending, drop a token when the
    cumulative probability before it exceeds p (the mask shifted by one keeps the first token).  True = kept, in index order."""
    sp, si = torch.sort(probs, descending=True)
    drop = torch.cumsum(sp, 0) > p
    drop = torch.cat([torch.zeros(1, dtype=torch.bool), drop[:-1]])
    keep = torch.zeros_like(drop)
    keep[si] = ~drop
    return keep


@pytest.mark.parametrize("T,p", [(0.6, 0.9), (1.0, 0.5), (2.0, 0.95), (0.3, 0.2), (1.0, 0.0), (1.0, 0.99)])
def test_keep_set_matches_reference_when_distinct(T, p):
    rng = np.random.default_rng(int(T * 100 + p * 10))
    checked = 0
    for _ in range(20):
        logits = (rng.standard_normal(3000) * 3).astype(np.float32)
        w = R.weights_fp64(logits, T)
        W = R.fixed_point(w)
        keep = R.keep_mask(W, R.nucleus_threshold(p, int(W.sum())))
        probs = torch.from_numpy(w / w.sum())
        # skip a draw whose threshold lies within rounding of a cumulative boundary (neither rule is defined to 1e-9 there)
        cums = np.cumsum(np.sort(w / w.sum())[::-1])
        if np.abs(cums - np.float32(p)).min() < 1e-9:
            continue
        assert np.array_equal(keep, reference_mask(probs, float(np.float32(p))).numpy())
        checked += 1
    assert checked >= 15


def test_tied_threshold_is_definite():
    """Four tied tokens and p = 0.5: the reference's sort leaves the kept three unspecified; the contract keeps the three lowest
    indices, and breaking ties by the higher index keeps the other three."""
    W = np.array([0, 5, 5, 5, 5, 1], dtype=np.int64) << 38
    thr = R.nucleus_threshold(0.5, int(W.sum()))
    assert np.nonzero(R.keep_mask(W, thr))[0].tolist() == [1, 2, 3]
    assert np.nonzero(R.keep_mask(W, thr, "ties_high"))[0].tolist() == [2, 3, 4]


def test_edges_of_p():
    W = np.array([3, 9, 9, 1, 0], dtype=np.int64) << 30
    assert R.keep_mask(W, R.nucleus_threshold(0.0, int(W.sum()))).tolist() == [False, True, False, False, False]
    assert R.keep_mask(W, R.nucleus_threshold(1.0, int(W.sum()))).all()


def test_draw_is_in_index_order():
    """The running kept sum in index order first exceeds the target at the token: a target in [0, W_0) draws token 0 even when
    token 0 is not the largest."""
    W = np.array([2, 7, 1], dtype=np.int64) << 40
    for r, want in ((0, 0), ((2 << 64) // 10 - 1, 0), ((2 << 64) // 10 + 1, 1), ((1 << 64) - 1, 2)):
        assert R.sample_from_weights(W, 1.0, r)[0] == want


# ---- named mistakes -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mistake", ["sorted_draw", "inclusive", "ties_high", "target32"])
def test_named_mistake_breaks_the_rule(mistake):
    """Each wrong rule gives a different token (or keep set) than the contract on some of 64 seeded draws of tied, peaked rows."""
    rng = np.random.default_rng(3)
    differ = 0
    for off in range(64):
        logits = np.round(rng.standard_normal(500) * 2).astype(np.float32)   # integers: many exact ties
        W = R.fixed_point(R.weights_fp64(logits, 1.0))
        r = R.draw_word(11, off, 0)
        good = R.sample_from_weights(W, 0.7, r)
        bad = R.sample_from_weights(W, 0.7, r, mistake)
        differ += good[0] != bad[0] or not np.array_equal(good[2], bad[2])
    assert differ > 0, f"{mistake} was not told apart from the contract"


def test_invalid_and_greedy_rows():
    l = np.array([1.0, 3.0, 3.0, -np.inf], dtype=np.float32)
    assert R.sample_row(l, 0.0, 0.9, 0, 0, 0) == (1, (0, 0, 0, 1, 0))
    assert R.sample_row(l, float("nan"), 0.9, 0, 0, 0)[0] == 1
    for bad in ([np.nan, 1.0], [np.inf, 1.0], [-np.inf, -np.inf]):
        assert R.sample_row(np.array(bad, dtype=np.float32), 1.0, 0.9, 0, 0, 0) == (0, (0, 0, 0, 0, 0))


def test_fixed_point_sum_fits():
    """The max weight is 1, so S < V 2^40 + 1 fits an int64 at any vocabulary the kernel takes (V <= 409 600)."""
    assert 409600 * 2 ** 40 < 2 ** 63
    W = R.fixed_point(np.ones(409600))
    assert int(W.sum()) == 409600 << 40


def test_weight_bound_grows_with_the_argument():
    l = np.array([0.0, -1.0, -50.0, -np.inf], dtype=np.float32)
    rel = R.weight_rel_bound(l, 0.5)
    assert rel[0] == 2.0 ** -21 and rel[1] < rel[2] and rel[3] == 2.0 ** -21


# ---- the C ABI and the wrapper --------------------------------------------------------------------------------------------------
def _aux_prototype(name):
    text = re.sub(r"/\*.*?\*/", "", open(N.AUX_HEADER_PATH).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)", text)
    assert m, f"{name} not declared"
    return [p.strip() for p in m.group(1).split(",")]


def test_binding_matches_header():
    params = _aux_prototype("mpig_aux_sample")
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
    res, args = N._AUX_SIGNATURES["mpig_aux_sample"]
    assert res is ctypes.c_int and args == want
    assert [re.sub(r".*\W", "", p) for p in params] == [
        "logits", "B", "V", "ld", "temperature", "top_p", "seed", "offset", "ids_out", "ids_stride", "tokens_out", "count", "done",
        "max_new", "eos_ids", "n_eos", "status", "debug", "debug_w", "stream"]
    assert "mpig_aux_sample_occupancy" in N._AUX_SIGNATURES


def _args(B=4, V=100):
    return dict(logits=torch.zeros((B, V)), temperature=torch.ones(B), top_p=torch.ones(B), offset=torch.zeros(1, dtype=torch.int64))


def test_wrapper_accepts():
    ids, max_new, eos = check_sample_args(**_args())
    assert ids.shape == (4,) and ids.dtype == torch.int64 and max_new == 0 and eos == []
    a = _args()
    a["logits"] = torch.zeros((4, 128))[:, :100]   # strided rows
    ids, max_new, eos = check_sample_args(**a, ids_out=torch.zeros((4, 1), dtype=torch.int64), tokens_out=torch.zeros((4, 7), dtype=torch.int32),
                                          count=torch.zeros(4, dtype=torch.int32), done=torch.zeros(4, dtype=torch.int32),
                                          eos_token_ids=range(8), status=torch.zeros(1, dtype=torch.int32),
                                          debug=torch.zeros((4, 5), dtype=torch.int64), debug_w=torch.zeros((4, 100)))
    assert max_new == 7 and eos == list(range(8))


@pytest.mark.parametrize("what", ["logits_dtype", "logits_rank", "logits_cols_strided", "empty", "temperature_shape", "top_p_dtype",
                                  "offset_dtype", "offset_size", "eos_count", "tokens_without_count", "count_without_tokens",
                                  "tokens_dtype", "ids_dtype", "ids_rows", "status_shape", "debug_shape", "debug_w_dtype"])
def test_wrapper_refusals(what):
    a = _args()
    kw = {}
    if what == "logits_dtype":
        a["logits"] = a["logits"].half()
    elif what == "logits_rank":
        a["logits"] = a["logits"].reshape(-1)
    elif what == "logits_cols_strided":
        a["logits"] = torch.zeros((4, 200))[:, ::2]
    elif what == "empty":
        a["logits"] = torch.zeros((4, 0))
    elif what == "temperature_shape":
        a["temperature"] = torch.ones(3)
    elif what == "top_p_dtype":
        a["top_p"] = a["top_p"].double()
    elif what == "offset_dtype":
        a["offset"] = torch.zeros(1, dtype=torch.int32)
    elif what == "offset_size":
        a["offset"] = torch.zeros(2, dtype=torch.int64)
    elif what == "eos_count":
        kw["eos_token_ids"] = list(range(MAX_EOS_IDS + 1))
    elif what == "tokens_without_count":
        kw["tokens_out"] = torch.zeros((4, 7), dtype=torch.int32)
    elif what == "count_without_tokens":
        kw["count"] = torch.zeros(4, dtype=torch.int32)
        kw["done"] = torch.zeros(4, dtype=torch.int32)
    elif what == "tokens_dtype":
        kw.update(tokens_out=torch.zeros((4, 7), dtype=torch.int64), count=torch.zeros(4, dtype=torch.int32),
                  done=torch.zeros(4, dtype=torch.int32))
    elif what == "ids_dtype":
        kw["ids_out"] = torch.zeros(4, dtype=torch.int32)
    elif what == "ids_rows":
        kw["ids_out"] = torch.zeros(5, dtype=torch.int64)
    elif what == "status_shape":
        kw["status"] = torch.zeros(2, dtype=torch.int32)
    elif what == "debug_shape":
        kw["debug"] = torch.zeros((4, 4), dtype=torch.int64)
    elif what == "debug_w_dtype":
        kw["debug_w"] = torch.zeros((4, 100), dtype=torch.float64)
    with pytest.raises(N.MagicPigError):
        check_sample_args(**a, **kw)


# ---- the runner: shapes and generate()'s arguments ------------------------------------------------------------------------------
def test_shape_eos_field():
    assert LLAMA31_8B.eos_token_ids == (128001, 128008, 128009)
    assert LLAMA31_70B.num_hidden_layers == 80 and LLAMA31_70B.rms_norm_eps == 1e-5 and LLAMA31_70B.eos_token_ids == LLAMA31_8B.eos_token_ids
    assert LlamaShape("tiny", 2, 512, 1024, 4, 2, 1000, 500000.0, 1e-5, (7,)).eos_token_ids == (7,)


def test_per_request():
    assert per_request(0.6, 3, "t") == [0.6] * 3
    assert per_request([0.1, 0.2], 2, "t") == [0.1, 0.2]
    assert per_request(torch.tensor([1.0, 2.0]), 2, "t") == [1.0, 2.0]
    with pytest.raises(ValueError):
        per_request([0.1, 0.2], 3, "t")


def test_generate_prompts():
    p = torch.arange(100)
    ps, shared = generate_prompts(p, 3, 1)
    assert shared and len(ps) == 3 and ps[0] is p
    ps, shared = generate_prompts(p[None], 2, 2)
    assert shared and ps[0].shape == (100,)
    ps, shared = generate_prompts([p, p[:80]], 2, 2)
    assert not shared and [x.numel() for x in ps] == [100, 80]
    with pytest.raises(ValueError):
        generate_prompts([p, p], 2, 1)   # different prompts need a context each
    with pytest.raises(ValueError):
        generate_prompts([p], 2, 2)
    with pytest.raises(ValueError):
        generate_prompts(torch.zeros((2, 5)), 2, 2)


def _gen_args(**kw):
    a = dict(lengths=[300], max_new_tokens=40, check_every=16, eos=(1, 2), max_length=512, num_sink=4, num_local=64, chunk_size=8192,
             generation_buffer=16, can_spill=True)
    a.update(kw)
    return a


def test_generate_args_accepted():
    check_generate_args(**_gen_args())
    check_generate_args(**_gen_args(lengths=[300, 472], max_new_tokens=40))   # 472 + 40 = max_length
    check_generate_args(**_gen_args(can_spill=False, max_new_tokens=17))      # 16 replays fit the window


@pytest.mark.parametrize("kw", [dict(max_new_tokens=0), dict(check_every=0), dict(eos=tuple(range(9))), dict(lengths=[473]),
                                dict(lengths=[300, 600]), dict(lengths=[68]), dict(chunk_size=0), dict(can_spill=False)])
def test_generate_args_refused(kw):
    with pytest.raises(ValueError):
        check_generate_args(**_gen_args(**kw))
