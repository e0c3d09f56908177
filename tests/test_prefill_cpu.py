"""Prefill without a GPU: the chunk bounds and prompt-length checks of LlamaDecodeRunner.prefill, the refusals of
LSHSparseAttnServer.prefill_attention, the ctypes binding of mpig_prefill_attend against the header, the reference's FlashInfer call
binding on prefill_attention, and the batched skipped-rescale restatement of tests/support/prefill_cases.py."""
import ctypes
import inspect
import math
import re

import pytest
import torch

from magicpig_b200 import _native as N
from magicpig_b200.attnserver import LSHSparseAttnServer, check_prefill_args
from magicpig_b200.llama_runner import plan_prefill_chunks
from tests.support.fp64 import softmax_state
from tests.support.prefill_cases import PF_KT, Case, check_rows, skip_rescale_rows, tokens_per_block


# ---- LlamaDecodeRunner.prefill: chunk bounds and prompt lengths ----------------------------------------------------------------
def test_chunks_of_the_bench_prompt():
    """98 000 tokens in chunks of 8 192: 11 whole chunks and a last one of 7 888 (llama.py:310-313)."""
    ch = plan_prefill_chunks(98000, 8192, 4, 64, 98304)
    assert len(ch) == 12 and ch[0] == (0, 8192) and ch[-1] == (90112, 98000)
    assert ch[-1][1] - ch[-1][0] == 7888
    assert all(b == a2 for (_, b), (a2, _) in zip(ch, ch[1:]))


@pytest.mark.parametrize("P,chunk,want", [(3000, 1024, [(0, 1024), (1024, 2048), (2048, 3000)]), (2048, 1024, [(0, 1024), (1024, 2048)]),
                                          (69, 8192, [(0, 69)]), (1025, 1024, [(0, 1024), (1024, 1025)])])
def test_chunk_bounds(P, chunk, want):
    assert plan_prefill_chunks(P, chunk, 4, 64, 4096) == want


@pytest.mark.parametrize("P,chunk", [(68, 1024), (10, 1024), (4097, 1024), (100, 0)])
def test_prompt_refused(P, chunk):
    """P <= sink + local (nothing to sample), P > max_length and a chunk size below 1 are refused before anything runs."""
    with pytest.raises(ValueError):
        plan_prefill_chunks(P, chunk, 4, 64, 4096)


# ---- LSHSparseAttnServer.prefill_attention: refusals ----------------------------------------------------------------------------
def _qkv(q_len=8, kv_len=12, Hq=32, Hkv=8, dtype=torch.bfloat16):
    return (torch.zeros((q_len, Hq, 128), dtype=dtype), torch.zeros((kv_len, Hkv, 128), dtype=dtype),
            torch.zeros((kv_len, Hkv, 128), dtype=dtype))


def test_prefill_args_accepted():
    for dt in (torch.bfloat16, torch.float16, torch.float32):
        check_prefill_args(*_qkv(dtype=dt), 32, 8, 128)
    check_prefill_args(*_qkv(12, 12), 32, 8, 128, causal=True, kv_layout="NHD")


@pytest.mark.parametrize("what", ["non_causal", "HND", "q_heads", "kv_heads", "head_dim", "v_shape", "q_rank", "q_longer", "empty",
                                  "int_dtype", "f64_dtype"])
def test_prefill_args_refused(what):
    q, k, v = _qkv()
    kw = {}
    if what == "non_causal":
        kw["causal"] = False
    elif what == "HND":
        kw["kv_layout"] = "HND"
    elif what == "q_heads":
        q = torch.zeros((8, 16, 128), dtype=torch.bfloat16)
    elif what == "kv_heads":
        k = v = torch.zeros((12, 4, 128), dtype=torch.bfloat16)
    elif what == "head_dim":
        q, k, v = q[..., :64], k[..., :64], v[..., :64]
    elif what == "v_shape":
        v = v[:11]
    elif what == "q_rank":
        q = q.reshape(8, 32 * 128)
    elif what == "q_longer":
        q, k, v = _qkv(13, 12)
    elif what == "empty":
        q = q[:0]
    elif what == "int_dtype":
        q = q.to(torch.int32)
    elif what == "f64_dtype":
        k = k.double()
    with pytest.raises(ValueError):
        check_prefill_args(q, k, v, 32, 8, 128, **kw)


# the keywords of the reference's prefill call (models/llama.py:250-257)
REFERENCE_CALL = dict(q="query_states", k="self.k_cache[:end]", v="self.v_cache[:end]", causal=True, allow_fp16_qk_reduction=True,
                      kv_layout="NHD")


def test_reference_call_binds():
    """The reference's flashinfer.prefill.single_prefill_with_kv_cache(...) keywords bind on prefill_attention, so llama.py changes
    one name only."""
    sig = inspect.signature(LSHSparseAttnServer.prefill_attention)
    bound = sig.bind(None, **REFERENCE_CALL)
    assert set(bound.arguments) == {"self", *REFERENCE_CALL}
    assert sig.parameters["causal"].default is True and sig.parameters["kv_layout"].default == "NHD"


# ---- the C ABI -------------------------------------------------------------------------------------------------------------------
def _prototype(name):
    text = re.sub(r"/\*.*?\*/", "", open(N.HEADER_PATH).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)", text)
    assert m, f"{name} not declared"
    return [p.strip() for p in m.group(1).split(",")]


def test_binding_matches_header():
    params = _prototype("mpig_prefill_attend")
    want = []
    for p in params:
        if "*" in p:
            want.append(ctypes.c_void_p)
        else:
            assert re.match(r"int\s+\w+$", p), p
            want.append(ctypes.c_int)
    res, args = N._SIGNATURES["mpig_prefill_attend"]
    assert res is ctypes.c_int and args == want
    assert [re.sub(r".*\W", "", p) for p in params] == ["ctx", "q_bf16", "k_bf16", "v_bf16", "q_len", "kv_len", "out_bf16",
                                                         "out_f32", "stream"]


# ---- the restatement itself ------------------------------------------------------------------------------------------------------
def test_batched_skip_rescale_matches_softmax_state():
    """skip_rescale_rows is fp64.softmax_state(skip_rescale=True) over 128-key tiles, row by row (masked keys at the end)."""
    g = torch.Generator().manual_seed(5)
    z = torch.randn((6, 700), generator=g, dtype=torch.float64) * 3
    z[:, 300] += 9.0
    z[2, 650:] = -math.inf
    V = torch.randn((700, 16), generator=g, dtype=torch.float64)
    got = skip_rescale_rows(z, V)
    for r in range(6):
        want, _ = softmax_state(z[r], V, skip_rescale=True, tile=PF_KT)
        assert torch.allclose(got[r], want, rtol=1e-12, atol=1e-12)


def test_check_rows_cover_block_edges():
    rows = check_rows(98000, 4, n_random=16)
    tb = tokens_per_block(4)
    assert tb == 32 and int(rows[0]) == 0 and int(rows[-1]) == 97999
    s = set(rows.tolist())
    assert all(m * tb in s and min(m * tb + tb - 1, 97999) in s for m in range(0, 98000 // tb + 1) if m * tb < 98000)


@pytest.mark.parametrize("regime", ["mean", "sinks", "sharp"])
def test_small_case_perturbations_move(regime):
    """A ragged case off every tile edge: each named perturbation moves the fp64 output by >= 10x the bar (CPU, fp64)."""
    c = Case(regime, 33, 257, Hq=28, Hkv=4, seed=3, dev="cpu")
    _, moved = c.check_inputs()
    assert set(moved) == {"limit_plus_1", "limit_minus_1", "drop_last_tile", "skip_rescale", "top_left", "head_mod"}
