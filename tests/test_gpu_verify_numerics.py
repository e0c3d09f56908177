"""Verification and tree steps against fp64 at the shapes the verification and tree lines measure (`-m gpu`).

Those lines run one request (B = 1) with Llama-3.1-8B heads (Hq 32, Hkv 8), K10 L150 over a 98 000-token prompt, in one context
with layer 1 sparse (n = 97 932 stored keys, M = 98 304, generation_buffer 256) and layer 0 dense (a full per-request cache of the
98 000 prompt rows), verification steps of up to 8 tokens, a window of NS + NL = 68 filled rows before the step.  Checked:

  * the path: the fused T-token kernel, 1, 1, 2, 2, 2 cluster waves at T = 2, 4, 7 (binary tree), 8 (chain), 8 (star tree);
  * sparse steps -- chains of 2, 4 and 8 tokens, the binary_depth3 tree (T = 7, G = 4) and the star_1+7 tree, fused_kreg 0 and 1,
    one T = 8 chain over a full 324-row window -- run with save_mask = 0 as the lines run them, codes and lists from a
    save_mask = 1 twin: query codes, nnz and index lists exact, every head's fp32 output within 1e-3 of the restatement under
    the step's causal or ancestor mask, the bf16 output the fp32 output rounded once, half-up;
  * dense steps: chains T = 2, 4, 5, 6, 7, 8 (T * G = 8 ... 32 query rows per kv-group: hi/lo packed, one m-tile, a second
    m-tile with 4 ... 16 real rows), and the two trees, against fp64 over the 98 000 prompt rows and the visible step rows;
  * accept and rewind on both layers: binary_depth3 then path [0, 2, 5], star_1+7 then [0, 7], the comb tree
    [-1, 0, 0, 2, 3, 4, 5, 6] then [0, 2, 3, 4, 5, 6, 7] (six rows move), star_1+7 then count = 0, a T = 8 chain then
    rewind(3); then a T = 1 step and a T = 2 chain on both layers against fp64 over the state the commit should leave -- the
    window plus the committed rows in path order, centred as the append centres them; the prompt rows plus the committed rows.

Regimes (test_gpu_batch_numerics.py's generator, each regime's 98 K store drawn once): R1 key mean, R2 sinks (the window holds
>= 90 % of the mass), R4 large logits with one dominant row -- the last stored key or the last window row; dense R2 and R4 with
the dominant row first, last or new.  Before any library call each case checks that its perturbations move the fp64 output by
>= 10x the bar: the regime's own; for R2 trees `tree_as_chain` (the ancestor mask read as a chain); for the steps after an
accept or rewind, the wrong commits that differ from the right one: `node_order` (nodes 0 .. count - 1), `path_dropped`
(nothing) and `step_kept` (every node).  Masks and commits are checked under R2 only: under R1 and R4 the step's own rows carry
too little of the mass for a wrong mask to show.  tests/test_verify_numerics_inputs_cpu.py runs the same generators and
self-checks without a GPU at a reduced size.
"""
import pytest
import torch

from magicpig_b200 import synth
from tests.support.fp64 import BAR, assert_rounded_half_up, rel_rows
from tests.support.library import DEV, NL, NS, d, skip_unless_132_sms, two_layer_context
from tests.support.sparse_cases import (ACCEPT_IDS, ACCEPTS, GEN, HKV, HQ, KK, LINE_TREES, LL, M_C2, N_C2, check_after,
                                        check_codes_lists, check_dense_after, check_inputs, check_outputs, dense_moves,
                                        fill_case, make_batch, make_dense, restate_dense, seed_of, step, twin_lists, twin_step)

pytestmark = pytest.mark.gpu
P = 98000
W = NS + NL                                      # filled window rows before the step
TREES = LINE_TREES
AFTER = (1, 2)                                   # the steps after an accept or rewind: T = 1, then a T = 2 chain


# ------------------------------------------------------------------------------------------------
# cases and the line's context
# ------------------------------------------------------------------------------------------------
_BASE = {}


def base_case(regime):
    """The 98 K store of the regime, drawn once (R4: without a dominant key)."""
    if regime not in _BASE:
        _BASE[regime] = make_batch(regime, 1, n=N_C2, lens=(NS + 8,), place="win", seed=seed_of("verify", regime))
    return _BASE[regime]


def sparse_inputs(label, regime, T, parents=None, place="key", lens=None):
    return make_batch(regime, 1, n=N_C2, T=T, lens=lens or (W + T,), place=place, seed=seed_of(label), parents=parents,
                      base=base_case(regime))


def line_ctx(save_mask, kreg=0, c=None, dense=None):
    """The lines' context: B = 1, layer 1 sparse (case c's store and window, or a small store), layer 0 dense (the dense case's
    prompt), verification steps of up to 8 tokens."""
    hf = c["hf"] if c is not None else synth.make_hash_func(d, KK, LL, seed=1)
    ctx = two_layer_context(KK, LL, HQ, HKV, 1, M_C2, GEN, hf, dict(decode_impl=1, fused_kreg=kreg, save_mask=save_mask,
                            out_f32=1), max_query_tokens=8, alloc_dense_kv=True)
    if c is not None:
        fill_case(ctx, c)
    else:
        g = torch.Generator(device=DEV).manual_seed(1)
        key = torch.randn((HKV, 300, d), generator=g, device=DEV).bfloat16()
        ctx.attn_fill(1, 0, key, key, key.float().norm(dim=-1))
        ctx.lsh_build(1, 0, ctx.hash_keys(key))
        ctx.window_fill(1, 0, torch.zeros((HKV, d), dtype=torch.bfloat16, device=DEV), key[:, :W].contiguous(),
                        key[:, :W].contiguous())
    if dense is not None:
        ctx.dense_fill(0, 0, dense["dk"][0].contiguous(), dense["dv"][0].contiguous(), dense["P"])
    return ctx


def plan(ctx, T, parents=None):
    ctx.plan(T, parents=None if parents is None else torch.tensor(parents, dtype=torch.int32, device=DEV))


def moves(label, moved):
    print(f"{label}: perturbations move the output by " + ", ".join(f"{k} {v:.2e}" for k, v in moved.items()))


# ---- 1. the path -------------------------------------------------------------------------------------------------------------
PATH_STEPS = [(2, None, 1), (4, None, 1), (7, TREES["binary_depth3"], 2), (8, None, 2), (8, TREES["star_1+7"], 2)]


def test_verify_path(cuda_lib):
    """The fused T-token kernel at every verification shape, in the cluster waves of a 132-SM H100."""
    skip_unless_132_sms()
    ctx = line_ctx(1)
    g = torch.Generator(device=DEV).manual_seed(2)
    for T, parents, waves in PATH_STEPS:
        q = torch.randn((1, T, HQ, d), generator=g, device=DEV).bfloat16()
        kv = torch.randn((1, T, HKV, d), generator=g, device=DEV).bfloat16()
        plan(ctx, T, None if parents is None else [parents])
        ctx.decode_tokens(1, T, q, kv, kv)
        got = (ctx.get_info("last_decode_fused"), ctx.get_info("tokens_cluster_waves"))
        print(f"T = {T} {'tree' if parents else 'chain'}: (last_decode_fused, tokens_cluster_waves) = {got}")
        assert got == (1, waves), f"T = {T}: {got}"
        if parents is None:
            ctx.rewind(torch.full((1,), T, dtype=torch.int32, device=DEV))
        else:
            ctx.accept(torch.zeros((1, T), dtype=torch.int32, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV))
    assert ctx.error_flags() == 0


# ---- 2. sparse steps ---------------------------------------------------------------------------------------------------------
# (label, regime, T, tree, fused_kreg, place, window rows after the step)
SPARSE = ([(f"T{T} {r}", r, T, None, 0, "key", None) for T in (2, 4, 8) for r in ("R1", "R2", "R4")]
          + [("T2 R1 kreg1", "R1", 2, None, 1, "key", None), ("T8 R4 kreg1", "R4", 8, None, 1, "key", None),
             ("T8 R2 full window", "R2", 8, None, 0, "key", NS + NL + GEN)]
          + [(f"{t} R2 kreg{k}", "R2", len(TREES[t]), t, k, "key", None) for t in TREES for k in (0, 1)]
          + [(f"{t} R4win", "R4", len(TREES[t]), t, 0, "win", None) for t in TREES])


@pytest.mark.parametrize("label,regime,T,tree,kreg,place,rows", SPARSE, ids=[s[0].replace(" ", "-") for s in SPARSE])
def test_sparse_step(cuda_lib, label, regime, T, tree, kreg, place, rows):
    parents = None if tree is None else [TREES[tree]]
    c = sparse_inputs(label, regime, T, parents, place, None if rows is None else (rows,))
    moves(label, check_inputs(c, parents, extra=("tree_as_chain",) if tree and regime == "R2" else ()))
    r = twin_step(lambda save_mask: line_ctx(save_mask, kreg, c), c, label, parents)
    check_outputs(c, r, check_codes_lists(c, r), label, parents)


# ---- 3. dense steps ----------------------------------------------------------------------------------------------------------
DENSE = ([(f"T{T} {r}{p}", r, T, None, p) for T in (2, 4, 5, 6, 7, 8) for r, p in (("R2", ""), ("R4", "first"), ("R4", "last"),
                                                                                       ("R4", "new"))]
         + [(f"{t} R2", "R2", len(TREES[t]), t, "") for t in TREES])


def dense_run(ctx, dn, label, parents=None):
    """Layer 0's step of dense case dn on ctx (planned) against fp64; returns the largest relative head error."""
    T = dn["q"].shape[1]
    if T == 1:
        out = ctx.dense_decode(0, dn["q"][:, 0].contiguous(), dn["k"][:, 0].contiguous(), dn["v"][:, 0].contiguous())
    else:
        out = ctx.dense_decode_tokens(0, T, dn["q"].contiguous(), dn["k"].contiguous(), dn["v"].contiguous())
    o32 = ctx.last_out_f32()
    worst = rel_rows(o32.reshape(1, T, HQ, d), restate_dense(dn, parents))
    print(f"{label}: largest relative head error {worst:.2e} ({worst / BAR:.1%} of the bar)")
    assert worst <= BAR, f"{label}: fp32 output differs from fp64 by {worst:.3e} relative (bar {BAR:g})"
    assert_rounded_half_up(out, o32, label)
    return worst


@pytest.mark.parametrize("label,regime,T,tree,place", DENSE, ids=[s[0].replace(" ", "-") for s in DENSE])
def test_dense_step(cuda_lib, label, regime, T, tree, place):
    parents = None if tree is None else [TREES[tree]]
    dn = make_dense(regime, 1, HQ, HKV, P, T, seed=seed_of("dense", label), place=place or "last", dev=DEV)
    moves(f"dense {label}", dense_moves(dn, parents, ("tree_as_chain",) if tree else ())[1])
    ctx = line_ctx(1, dense=dn)
    plan(ctx, T, parents)
    dense_run(ctx, dn, f"dense {label}", parents)
    assert ctx.error_flags() == 0


# ---- 4. accept and rewind ----------------------------------------------------------------------------------------------------


def both_layers(ctxs, c, dn, parents, label):
    """One step of the sparse case c and the dense case dn on both layers of ctxs = (save_mask 0, save_mask 1 twin), checked
    against fp64."""
    rs = []
    for save_mask, ctx in enumerate(ctxs):
        rs.append(step(ctx, c, parents, lists=bool(save_mask)))
        dense_run(ctx, dn, f"{label} dense (save_mask {save_mask})", parents)
    r = twin_lists(rs[0], rs[1], label)
    assert r["fused"] == 1, f"{label}: last_decode_fused = {r['fused']}"
    check_outputs(c, r, check_codes_lists(c, r), f"{label} sparse", parents)


@pytest.mark.parametrize("label,tree,path", ACCEPTS, ids=ACCEPT_IDS)
def test_accept_then_steps(cuda_lib, label, tree, path):
    """A tree step and accept(path), or a chain step and rewind(3), on both layers; then a T = 1 step and a T = 2 chain against
    fp64 over what the commit should leave."""
    T = 8 if tree is None else len(tree)
    parents = None if tree is None else [tree]
    keep = [path]
    c = sparse_inputs(label, "R2", T, parents)
    dn = make_dense("R2", 1, HQ, HKV, P, T, seed=seed_of("dense", label), dev=DEV)
    extra = ("tree_as_chain",) if tree else ()
    moves(f"{label} step sparse", check_inputs(c, parents, extra=extra))
    moves(f"{label} step dense", dense_moves(dn, parents, extra)[1])
    seed = seed_of("after", label)
    nxt, moved = check_after(c, keep, AFTER, seed)
    moves(f"{label} next sparse", moved)
    nxt_d, moved = check_dense_after(dn, keep, AFTER, seed + 100)
    moves(f"{label} next dense", moved)
    ctxs = (line_ctx(0, 0, c, dn), line_ctx(1, 0, c, dn))
    both_layers(ctxs, c, dn, parents, f"{label} step")
    for ctx in ctxs:
        if tree is None:
            ctx.rewind(torch.tensor([T - len(path)], dtype=torch.int32, device=DEV))
        else:
            ctx.accept(torch.tensor([path + [0] * (T - len(path))], dtype=torch.int32, device=DEV),
                       torch.tensor([len(path)], dtype=torch.int32, device=DEV))
    for x, xd, T2 in zip(nxt, nxt_d, AFTER):
        both_layers(ctxs, x, xd, None, f"{label} then T{T2}")
    for ctx in ctxs:
        assert ctx.error_flags() == 0
