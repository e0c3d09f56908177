"""The generator and self-checks of tests/test_gpu_config_numerics.py, without a GPU at a reduced size.

K11 L300 (two tag passes of 253 + 47 tables) over n = 20 000 keys cut into 4 segments, Hq 8 / Hkv 1 (one kv-group), 8 slots
holding different documents with ragged windows: every regime's property and every named perturbation -- the regime's own,
`window_of_request_0`, `wrong_document` over 8 slots, `drop_sampled`, `cross_pass`, `wrong_weights`, `drop_segment_s` and
`window_of_head_0` -- must move the fp64 output by >= 10x the 1e-3 bar, and keys that collide once in each pass must exist for
every head.
"""
import pytest

from tests.support.config_cases import REG_CHUNKS, check_config_inputs, chunk_streams, pass_sets, seg_bounds
from tests.support.fp64 import query_codes
from tests.support.sparse_cases import LENS, make_batch, perturbations

SMALL = dict(n=20000, dev="cpu", Hq=8, Hkv=1, K=11, L=300)
SEGS = seg_bounds(4, 20480)
_BASE = {}


def case(regime, place="key", dominant=None):
    if regime not in _BASE:
        _BASE[regime] = make_batch(regime, 8, C=8, place="win", lens=(12,), seed=11, **SMALL)
    return make_batch(regime, 8, C=8, place=place, dominant=dominant, seed=12, base=_BASE[regime], **SMALL)


@pytest.mark.parametrize("regime,place,seg", [("R1", "key", None), ("R2", "key", None), ("R4", "key", None),
                                              ("R4", "key", 1), ("R4", "win", None)],
                         ids=["R1", "R2", "R4last", "R4seg1", "R4win"])
def test_config_regime_is_sensitive(regime, place, seg):
    c = case(regime, place, None if seg is None else seg * SEGS[1])
    assert len({w.shape[1] for w in c["win_k"]}) == len(set(LENS)), "windows are not ragged"
    if regime == "R1" or place == "key" and regime == "R4":
        assert "wrong_document" in perturbations(c), "wrong_document is not checked over 8 slots"
    codes = check_config_inputs(c, SEGS, f"cpu {regime}{place}")
    _, cross = pass_sets(c, codes)
    assert int(cross.min()) > 0
    print(f"cpu {regime}{place}: keys hit once in each pass per head {int(cross.min())} .. {int(cross.max())}; longest chunk "
          f"stream {chunk_streams(c, codes, SEGS)} (registers hold {REG_CHUNKS})")


def test_chunk_streams_count_buckets():
    """chunk_streams against a direct count for one head: ceil(bucket keys of the segment / 32) summed over a pass."""
    c = case("R1")
    codes = query_codes(c["q"], c["hf"], c["K"], c["L"])[0]
    kc = c["slots"][0]["kcodes"][0]
    qc = codes[0, 0, 0]
    nseg, seg_len = SEGS
    want = 0
    for s in range(nseg):
        part = kc[:, s * seg_len:(s + 1) * seg_len]
        for p0 in (0, 253):
            want = max(want, sum(-(-int((part[t] == qc[t]).sum()) // 32) for t in range(p0, min(300, p0 + 253))))
    one = dict(c, B=1, slot_of=[0])
    got = chunk_streams(one, codes[:1, :, :1].expand(1, 1, 1, 300).contiguous(), SEGS)
    assert got == want
