"""The sparse layer against fp64 at BASELINE's other GPU configurations (`-m gpu`).

test_gpu_numerics.py, test_gpu_batch_numerics.py and test_gpu_chunk_numerics.py hold the decode kernels to fp64 at K <= 10,
L <= 150 and at most the C2 store.  This file does the same, with the generator and restatement of test_gpu_batch_numerics.py,
at the shapes of BASELINE.json's C3, C4 and C5:

  * C4      ProLong K11 L300 over n = 199 932 keys (M = 200 448), Hq 32 / Hkv 8: two tag passes of 253 + 47 tables in the fused
            kernel, uint16 probe tags on the three-launch path, compile-time weight exponents 11 and 299, key codes that straddle
            32-bit words in the key hash;
  * C4max   the same at n = 499 932 (M = 500 480), the size test_gpu_parity.py::test_full_size_properties uses;
  * C3      B = 8 over 8 slots of n = 32 700 keys (M = 33 024), one document per slot, ragged windows;
  * C5      the 70B model's per-rank shape under KV-head TP = 8: Hq 8, Hkv 1, n = 97 932 (M = 98 304), one group of 8 heads.

Every case draws its stores once per (shape, regime) (the fp64 key projections dominate the runtime), checks in fp64 that its
named perturbations move the output by >= 10x the 1e-3 bar, hashes the keys with the library (codes must equal the fp64 ones
except within SIMHASH_EPS x the mean key norm of a zero projection) and builds the tables from those codes, then holds query
codes, nnz, index lists, the fp32 output (per head, 1e-3 of max|fp64|) and the bf16 output (fp32 rounded half-up) to the
restatement.  The perturbations added here: `cross_pass` (collision counts of the two tag passes never combined), `wrong_weights`
(the weight of K10 L150), `drop_segment_s` (the sampled keys of key segment s removed), `wrong_document` over 8 slots and
`window_of_head_0` (every head of the group takes head 0's window half).  Each C4 case also prints the largest number of
32-candidate chunks one CTA streams in one tag pass, computed from the codes and the segment bounds; some C4 case must exceed the
256 chunks a pass keeps in registers.  tests/test_config_numerics_inputs_cpu.py runs the generator and the self-checks without
a GPU at a reduced size.
"""
import gc
import os
import socket

import pytest
import torch

from magicpig_b200 import synth
from tests.support.config_cases import REG_CHUNKS, check_config_inputs, chunk_streams, seg_bounds
from tests.support.fp64 import SIMHASH_EPS
from tests.support.library import DEV, NL, NS, assert_tables_equal, d, lsh_tables, skip_unless_132_sms, two_layer_context
from tests.support.sparse_cases import (GEN, LENS, TREE, batch_ctx, check_codes_lists, check_outputs, make_batch, seed_of,
                                        step, twin_step)

pytestmark = pytest.mark.gpu

SHAPES = {
    "C4": dict(B=1, Hq=32, Hkv=8, K=11, L=300, n=199932, M=200448),
    "C4max": dict(B=1, Hq=32, Hkv=8, K=11, L=300, n=499932, M=500480),
    "C3": dict(B=8, Hq=32, Hkv=8, K=10, L=150, n=32700, M=33024),
    "C5": dict(B=1, Hq=8, Hkv=1, K=10, L=150, n=97932, M=98304),
}
# on a 132-SM H100: table_segments, fused_applicable, fused_cluster_waves, last_decode_fused of a single-token step
GEOMETRY = {
    "C4": (4, 1, 2, 1),       # clusters of 4 CTAs (1024 threads), two waves
    "C4max": (8, 1, 2, 1),    # clusters of 8 CTAs of 512 threads
    "C3": (1, 1, 1, 1),       # one 512-thread CTA per head, codes from the SimHash kernel
    "C5": (8, 1, 1, 1),       # 8 clusters of 8
}
# tokens_cluster_waves of a T-token step
TOKEN_WAVES = {("C4", 4): 3, ("C4", 8): 5, ("C5", 4): 2}


def slot_count(shape):
    return SHAPES[shape]["B"]   # C3: one document per request; the others: B = 1


def segments(shape):
    return seg_bounds(GEOMETRY[shape][0], SHAPES[shape]["M"])


def is_fused(shape):
    return bool(GEOMETRY[shape][3])


# ------------------------------------------------------------------------------------------------
# generator: one draw of the stores per (shape, regime)
# ------------------------------------------------------------------------------------------------
_BASE = {}
LONGEST = {}   # C4 case -> its largest chunk stream of one CTA in one tag pass


def base_case(shape, regime):
    """The stores of (shape, regime), drawn once and reused by every case of it (R4: without a dominant key)."""
    key = (shape, regime)
    if key not in _BASE:
        if shape == "C4max":   # 4 GB of fp64 draws and 5 GB of stores: never kept next to the others
            release()
        s = SHAPES[shape]
        _BASE[key] = make_batch(regime, s["B"], C=slot_count(shape), n=s["n"], lens=(NS + 8,), place="win",
                                seed=seed_of(shape, regime), Hq=s["Hq"], Hkv=s["Hkv"], K=s["K"], L=s["L"])
    return _BASE[key]


def release():
    _BASE.clear()
    gc.collect()
    torch.cuda.empty_cache()


def make_case(label, shape, regime, place="key", dominant=None, T=1, parents=None, lens=LENS):
    s = SHAPES[shape]
    return make_batch(regime, s["B"], C=slot_count(shape), n=s["n"], T=T, lens=lens, place=place, seed=seed_of(label),
                      Hq=s["Hq"], Hkv=s["Hkv"], K=s["K"], L=s["L"], parents=parents, dominant=dominant,
                      base=base_case(shape, regime))


# ------------------------------------------------------------------------------------------------
# the library's key codes
# ------------------------------------------------------------------------------------------------
def library_codes(c, impl=1):
    """Every slot's keys hashed by the library (keyhash_impl impl), checked against the fp64 codes: a code may differ only where
    one of its K projections is within SIMHASH_EPS x the mean key norm of zero (no count allowance)."""
    from magicpig_b200.ops import Context
    K, L = c["K"], c["L"]
    hasher = Context(K, L, 1, c["Hq"], c["Hkv"], d, 1, c["n"], device=DEV)
    hasher.set_option("keyhash_impl", impl)
    hasher.set_hash_func(c["hf"].contiguous())
    hfd = c["hf"].double()
    out = []
    for st in c["slots"]:
        ours = hasher.hash_keys(st["key"].contiguous())
        bad = torch.nonzero(ours != st["kcodes"])
        scale = float(st["key"].float().norm(dim=-1).mean())
        for i in range(0, bad.shape[0], 1 << 16):   # the fp64 projections of the differing (group, table, key) triples only
            part = bad[i:i + (1 << 16)]
            kk = st["key"][part[:, 0], part[:, 2]].double()
            cols = part[:, 1, None] * K + torch.arange(K, device=DEV)[None]
            margin = (hfd.t()[cols] * kk[:, None]).sum(-1).abs().min(dim=-1).values
            assert float(margin.max()) < SIMHASH_EPS * scale, \
                f"keyhash_impl {impl}: {bad.shape[0]} key codes differ, margin {float(margin.max()) / scale:.2e} of the key norm"
        out.append(ours)
    del hasher
    return out


def use_library_codes(c):
    for st, codes in zip(c["slots"], library_codes(c)):
        st["kcodes"] = codes


# ------------------------------------------------------------------------------------------------
# one case: self-checks, the library's codes, the runs
# ------------------------------------------------------------------------------------------------
def run_path(c, shape, label, kreg=0, impl=1, parents=None, ctx_hook=None):
    """One step of case c on the path the shape runs (impl 0: the three-launch path), checked against fp64.  Fused steps run
    with save_mask = 0 and take codes and lists from a save_mask = 1 twin, which must sample the same counts."""
    s = SHAPES[shape]
    T = c["q"].shape[1]

    def make_ctx(save_mask):
        ctx = batch_ctx(c, C=0, M=s["M"], kreg=kreg, save_mask=save_mask, t_max=T)
        if impl == 0:
            ctx.set_option("decode_impl", 0)
        return ctx
    r = twin_step(make_ctx, c, label, parents, impl == 1 and (T > 1 or is_fused(shape)), ctx_hook)
    sets = check_codes_lists(c, r)
    worst = check_outputs(c, r, sets, label, parents)
    torch.cuda.empty_cache()
    return worst, r


def config_case(label, shape, regime, place="key", dominant=None, T=1, parents=None, lens=LENS, runs=((0, 1), (1, 1))):
    """Generate, self-check, switch to the library's key codes and run every (fused_kreg, decode_impl) of runs."""
    c = make_case(label, shape, regime, place, dominant, T, parents, lens)
    codes = check_config_inputs(c, segments(shape), label)
    if shape.startswith("C4"):
        longest = chunk_streams(c, codes, segments(shape))
        print(f"{label}: largest chunk stream of one CTA in one tag pass {longest} (registers hold {REG_CHUNKS})")
        LONGEST[label] = longest
    use_library_codes(c)
    for kreg, impl in runs:
        run_path(c, shape, f"{label} kreg{kreg}" + (" three-launch" if impl == 0 else ""), kreg, impl, parents)
    return c, codes


# ---- 1. path and geometry per shape ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", list(SHAPES))
def test_config_geometry(cuda_lib, shape):
    """table_segments, fused_applicable, fused_cluster_waves and last_decode_fused of a single-token step, and
    tokens_cluster_waves of T-token steps, on a 132-SM H100."""
    skip_unless_132_sms()
    s = SHAPES[shape]
    B, Hq, Hkv, K, L = s["B"], s["Hq"], s["Hkv"], s["K"], s["L"]
    for T in [1] + sorted(t for (sh, t) in TOKEN_WAVES if sh == shape):
        ctx = two_layer_context(K, L, Hq, Hkv, B, s["M"], GEN, max_query_tokens=T)
        got = [ctx.get_info("table_segments"), ctx.get_info("fused_applicable"), ctx.get_info("fused_cluster_waves")]
        g = torch.Generator(device=DEV).manual_seed(1)
        ctx.set_hash_func(synth.make_hash_func(d, K, L, seed=1).to(DEV))
        key = torch.randn((Hkv, 300, d), generator=g, device=DEV).bfloat16()
        for b in range(B):
            ctx.attn_fill(1, b, key, key, key.float().norm(dim=-1))
            ctx.lsh_build(1, b, ctx.hash_keys(key))
            ctx.window_fill(1, b, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=DEV), key[:, :NS + NL].contiguous(),
                            key[:, :NS + NL].contiguous())
        q = torch.randn((B, T, Hq, d), generator=g, device=DEV).bfloat16()
        kv = torch.randn((B, T, Hkv, d), generator=g, device=DEV).bfloat16()
        if T == 1:
            ctx.plan()
            ctx.decode(1, q[:, 0].contiguous(), kv[:, 0].contiguous(), kv[:, 0].contiguous())
            got.append(ctx.get_info("last_decode_fused"))
            print(f"{shape}: (table_segments, fused_applicable, fused_cluster_waves, last_decode_fused) = {tuple(got)}")
            assert tuple(got) == GEOMETRY[shape], f"{shape}: {tuple(got)}"
        else:
            ctx.plan(T)
            ctx.decode_tokens(1, T, q, kv, kv)
            w = ctx.get_info("tokens_cluster_waves")
            print(f"{shape} T={T}: tokens_cluster_waves = {w}")
            assert ctx.get_info("last_decode_fused") == 1 and w == TOKEN_WAVES[(shape, T)], f"{shape} T={T}: waves {w}"
        del ctx


# ---- 2. the key hash at full size --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("shape", ["C4", "C3", "C5"])
def test_config_key_hash(cuda_lib, shape, impl):
    """ctx.hash_keys (keyhash_impl 1: the persistent pipeline, 0: one tile per CTA) over every store of the shape against the
    fp64 codes of the same keys; at C4 a code of 11 bits straddles a 32-bit word of the projection row for some tables."""
    c = base_case(shape, "R1")
    library_codes(c, impl)


# ---- 3. C4 single-token -------------------------------------------------------------------------------------------------------
C4_SINGLE = [("R1", "key", None), ("R2", "key", None), ("R4", "key", None), ("R4", "key", 1), ("R4", "key", 3),
             ("R4", "win", None)]


@pytest.mark.parametrize("regime,place,seg", C4_SINGLE,
                         ids=["R1", "R2", "R4last", "R4seg1", "R4seg3", "R4win"])
def test_c4_single(cuda_lib, regime, place, seg):
    """C4, B = 1: fused_kreg 0 and 1, and the three-launch path (uint16 probe tags).  R4's dominant key is the last stored key,
    the first key of segment 1 or 3, or every request's last window row."""
    dominant = None if seg is None else seg * segments("C4")[1]
    config_case(f"C4 {regime}{place if seg is None else f'seg{seg}'}", "C4", regime, place, dominant,
                lens=(324,), runs=((0, 1), (1, 1), (0, 0)))


# ---- 4. C4 verification -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tree", [False, True], ids=["chain4", "tree8"])
def test_c4_verification(cuda_lib, tree):
    """A T = 4 chain (R4) or the 8-node tree (R2) at C4: the T-token instantiation, two tag passes, several waves."""
    T, parents = (8, [TREE]) if tree else (4, None)
    config_case(f"C4 {'tree8' if tree else 'T4'}", "C4", "R2" if tree else "R4", T=T, parents=parents, lens=(200,),
                runs=((0, 1), (1, 1)))


def test_c4_overflows_register_window(cuda_lib):
    """Some C4 case streams more chunks in one tag pass than the registers hold, so the per-pass overflow loops ran."""
    if not LONGEST:
        pytest.skip("no C4 case ran in this session")
    assert max(LONGEST.values()) > REG_CHUNKS, f"no C4 case exceeds {REG_CHUNKS} chunks in a pass: {LONGEST}"


# ---- 5. C4 spill --------------------------------------------------------------------------------------------------------------
def test_c4_spill(cuda_lib):
    """A full 324-row window at C4 spills 256 keys into segment 3: the tables equal a device rebuild over the stored keys, and a
    decode over the store as it now is matches fp64."""
    s = SHAPES["C4"]
    nseg, seg_len = segments("C4")
    c = make_case("C4 spill", "C4", "R1", lens=(NS + NL + GEN,))
    check_config_inputs(c, segments("C4"), "C4 before spill")
    use_library_codes(c)
    ctx = batch_ctx(c, C=0, M=s["M"], save_mask=1)
    r = step(ctx, c)
    check_outputs(c, r, check_codes_lists(c, r), "C4 before spill")
    st, n = c["slots"][0], c["n"]
    c["win_k"][0] = torch.cat([c["win_k"][0], (c["k_new"][0, 0] - st["avg"])[:, None]], dim=1)
    c["win_v"][0] = torch.cat([c["win_v"][0], c["v_new"][0, 0][:, None]], dim=1)
    assert c["win_k"][0].shape[1] == NS + NL + GEN
    g = GEN
    assert ctx.spill_window().tolist() == [g]
    assert (n // seg_len, (n + g - 1) // seg_len) == (nseg - 1, nseg - 1), "the spilled keys are not in the last segment"
    k_st, v_st, kn_st = ctx.read_cache(1)
    assert torch.equal(k_st[0, :, n:n + g].contiguous().view(torch.int16),
                       c["win_k"][0][:, NS:NS + g].contiguous().view(torch.int16)), "spilled keys"
    other = two_layer_context(c["K"], c["L"], c["Hq"], c["Hkv"], 1, s["M"], 8, c["hf"])
    new_codes = other.hash_keys(k_st[0, :, n:n + g].contiguous())
    other.lsh_build(1, 0, torch.cat([st["kcodes"], new_codes], dim=-1).contiguous())
    assert_tables_equal(lsh_tables(ctx, 1), lsh_tables(other, 1), [0])
    del other
    torch.cuda.empty_cache()
    # the store as it now is: the prompt, the spilled keys (the library's codes of them), the window's sinks and newest rows
    st.update(key=k_st[0, :, :n + g], value=v_st[0, :, :n + g], kn=kn_st[0, :, :n + g],
              kcodes=torch.cat([st["kcodes"], new_codes], dim=-1))
    c["n"] = n + g
    c["win_k"][0] = torch.cat([c["win_k"][0][:, :NS], c["win_k"][0][:, NS + g:]], dim=1)
    c["win_v"][0] = torch.cat([c["win_v"][0][:, :NS], c["win_v"][0][:, NS + g:]], dim=1)
    gq = torch.Generator(device=DEV).manual_seed(5)
    c["k_new"] = (torch.randn((1, 1, c["Hkv"], d), generator=gq, device=DEV, dtype=torch.float64)
                  + st["mu"].reshape(1, 1, c["Hkv"], d)).bfloat16()
    c["v_new"] = torch.randn((1, 1, c["Hkv"], d), generator=gq, device=DEV).bfloat16()
    r = step(ctx, c)
    assert r["fused"] == 1
    sets = check_codes_lists(c, r)
    check_outputs(c, r, sets, "C4 after spill")
    assert any(bool((x >= n).any()) for x in sets[0][0]), "no head sampled a spilled key"
    del ctx, k_st, v_st, kn_st


# ---- 6. C4max -----------------------------------------------------------------------------------------------------------------
def test_c4max_single(cuda_lib):
    """C4 at n = 499 932: one R1 single-token step on the path the library picks (8 segments of 62 592 keys)."""
    try:
        config_case("C4max R1", "C4max", "R1", lens=(324,), runs=((0, 1),))
    finally:
        release()


# ---- 7. C3 --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", ["R1", "R2", "R4"])
def test_c3(cuda_lib, regime):
    """B = 8, eight slots with one document each, ragged windows: every request against ITS slot's store and its window."""
    config_case(f"C3 {regime}", "C3", regime)


# ---- 8. C5 rank ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("regime,place", [("R1", "key"), ("R2", "key"), ("R4", "key"), ("R4", "win")],
                         ids=["R1", "R2", "R4key", "R4win"])
def test_c5_rank(cuda_lib, regime, place):
    """One kv-group of 8 heads (Hq 8, Hkv 1) over 8 segments of 12 288 keys."""
    config_case(f"C5 {regime}{place}", "C5", regime, place, lens=(324,))


def test_c5_rank_chain(cuda_lib):
    config_case("C5 T4", "C5", "R4", T=4, lens=(200,), runs=((0, 1), (1, 1)))


def test_c5_rank_allgather(cuda_lib):
    """PeerExchange.decode_allgather at world size 1 (the fused kernel stores the head outputs into the gather slot) equals
    decode's bf16 output bit for bit, on the C5 shape against fp64."""
    import torch.distributed as dist
    from magicpig_b200.peer import PeerExchange

    def allgather(ctx, r):
        own_pg = not dist.is_initialized()
        if own_pg:
            sk = socket.socket()
            sk.bind(("127.0.0.1", 0))
            os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(sk.getsockname()[1])
            sk.close()
            dist.init_process_group("gloo", rank=0, world_size=1)
        try:
            px = PeerExchange(ctx, 0, 1, c["Hq"] * d * 2)
            got = px.decode_allgather(1, c["q"][:, 0].contiguous(), c["k_new"][:, 0].contiguous(), c["v_new"][:, 0].contiguous())
            torch.cuda.synchronize()
            assert torch.equal(got.reshape(-1), r["out"].reshape(-1)), "decode_allgather differs from decode"
            px.close()
        finally:
            if own_pg:
                dist.destroy_process_group()

    c = make_case("C5 allgather", "C5", "R1", lens=(324,))
    check_config_inputs(c, segments("C5"), "C5 allgather")
    use_library_codes(c)
    run_path(c, "C5", "C5 allgather", ctx_hook=allgather)
