"""Model-shaped inputs of the sparse and dense decode layers, their self-checks and the GPU-side steps over them.

Two generators of sparse cases, both in the slot layout that support.fp64.restate reads (c["slots"], c["slot_of"], per-request
window lists):
  * make_case: test_gpu_numerics.py's regimes R1..R5, one slot per request, CPU tensors, tuned on the C oracle's query codes;
  * make_batch: test_gpu_batch_numerics.py's and test_gpu_config_numerics.py's batches of B requests on C slots at the measured
    shapes, ragged windows, tuned on fp64 query codes, on any device.
They draw different inputs on purpose and keep their own tuning.  Dense cases: make_dense (one prompt per request, or one for
all) and make_dense_slots (shared prefix, ragged tails).  next_case / next_dense turn an R2 case and the nodes its step commits
(an accepted path, a rewind) into the case of the next step; check_after / check_dense_after self-check such a sequence against
wrong commits (ACCEPT_VARIANTS).
"""
import math
import zlib

import torch

import oracle
from magicpig_b200 import synth
from tests.support.fp64 import (BAR, SIMHASH_EPS, assert_rounded_half_up, avg_of, centred, head_mask, key_codes, lsh_weight,
                                query_codes, rel_rows, restate, sample_sets, softmax_state, unit, visible)
from tests.support.library import DEV, NL, NS, d, two_layer_context

RD = math.sqrt(d)
SELF_CHECK = {"R1": "uncentred", "R2": "drop_newest", "R3": "ln_merge", "R4": "skip_rescale"}
TREE = [-1, 0, 0, 1, 1, 2, 3, 3]
# the tree line's trees (node t's parent), and its accept cases: (label, the step's tree -- None: a T = 8 chain --, the nodes
# committed in order: an accepted root path, or the 5 a rewind(3) keeps)
LINE_TREES = {"binary_depth3": [-1, 0, 0, 1, 1, 2, 2], "star_1+7": [-1] + [0] * 7}
COMB = [-1, 0, 0, 2, 3, 4, 5, 6]
ACCEPTS = [("binary_depth3 [0,2,5]", LINE_TREES["binary_depth3"], [0, 2, 5]),
           ("star_1+7 [0,7]", LINE_TREES["star_1+7"], [0, 7]),
           ("comb [0,2,3,4,5,6,7]", COMB, [0, 2, 3, 4, 5, 6, 7]),
           ("star_1+7 count 0", LINE_TREES["star_1+7"], []),
           ("T8 rewind 3", None, [0, 1, 2, 3, 4])]
ACCEPT_IDS = ["binary", "star", "comb", "star-none", "rewind"]
# the measured lines: Llama-3.1-8B heads, K10 L150, one 98 K-token context (C2)
HQ, HKV, KK, LL = 32, 8, 10, 150
N_C2, M_C2, M_LONG = 97932, 98304, 131072
GEN = 256
LENS = (69, 150, 324, 200)            # window rows after the step, cycled over the requests (324 = NS + NL + GEN: full)
EVERY_HEAD = {"drop_sampled"}   # perturbations that must move every checked head, not only the most sensitive one


def _terms(c, sets, b, t, h, win_extra=None):
    """Raw sampled scores s / sqrt(d), their LSH offsets -log(w + 1e-4), the window scores (filled rows, then win_extra) and
    the sample set of one head."""
    st, g = c["slots"][c["slot_of"][b]], h // c["G"]
    qh = c["q"][b, t, h].double()
    idx = sets[b][t][h]
    s = st["key"][g, idx].double() @ qh
    cs = s / (qh.norm() * st["kn"][g, idx].double())
    off = -torch.log(lsh_weight(cs, c["K"], c["L"]) + 1e-4)
    wk = c["win_k"][b][g] if win_extra is None else torch.cat([c["win_k"][b][g], win_extra])
    return s / RD, off, (wk.double() @ qh) / RD, idx


def _each_head(c):
    B, T, Hq = c["q"].shape[:3]
    return [(b, t, h) for b in range(B) for t in range(T) for h in range(Hq)]


# ------------------------------------------------------------------------------------------------
# make_case: one slot per request, regimes R1..R5
# ------------------------------------------------------------------------------------------------
def cpu_codes(c) -> torch.Tensor:
    """Query codes (B, T, Hq, L) of the C oracle's SimHash."""
    B, T, Hq = c["q"].shape[:3]
    codes, _ = oracle.simhash(c["q"].reshape(-1, d).contiguous(), c["hf"], c["K"], c["L"])
    return codes.reshape(B, T, Hq, c["L"])


def _set_stores(c, key, kn, kcodes):
    """Slot b's key, norms and codes: request b's rows of the (B, ...) tensors."""
    for b, st in enumerate(c["slots"]):
        st.update(key=key[b], kn=kn[b], kcodes=kcodes[b])


def _rehash(c):
    """Norms and codes of every slot's keys after an edit, computed over all slots at once as the generator first did."""
    key = torch.stack([st["key"] for st in c["slots"]])
    _set_stores(c, key, key.norm(p=2, dim=-1).float(), synth.hash_keys(key, c["hf"], c["K"], c["L"]))


def make_case(regime, B, Hq, Hkv, n, K, L, seed, T=1, place="last", parents=None):
    """Sparse-layer inputs of one regime (R1..R5, R4 with the dominant key `place`d first or last in the store), tuned on the
    CPU codes; request b on slot b.  CPU tensors: q (B,T,Hq,d); per slot key/value (Hkv,n,d) centred store, kn, avg (Hkv,d),
    kcodes; per request win_k/win_v (Hkv,NS+NL,d) centred window; k_new/v_new (B,T,Hkv,d) as the model produces them
    (uncentred)."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.randn(s, generator=g, dtype=torch.float64)   # noqa: E731
    G, W = Hq // Hkv, NS + NL
    hf = synth.make_hash_func(d, K, L, seed=seed + 1)
    u = unit(rnd, B, Hkv)                                                   # one direction per kv group
    qn = 0.5 if regime == "R4" else 1.0
    q = qn * torch.randn((B, T, Hq, d), generator=g, dtype=torch.float64) + RD * u.repeat_interleave(G, 1)[:, None]
    mu = torch.zeros((B, Hkv, 1, d), dtype=torch.float64)
    if regime == "R1":   # |mu| ~ 4 |noise|, partly along the queries (which is what makes an uncentred key visible)
        mu = 4.0 * (0.8 * torch.randn((B, Hkv, 1, d), generator=g, dtype=torch.float64) + 0.6 * RD * u[:, :, None])
    key = torch.randn((B, Hkv, n, d), generator=g, dtype=torch.float64)
    if regime != "R4":   # a share of the keys clusters around the group direction, so that K10 L150 samples some of them
        pull = (torch.rand((B, Hkv, n, 1), generator=g) < 0.125) * torch.rand((B, Hkv, n, 1), generator=g, dtype=torch.float64) * 1.2
        key = key + pull * RD * u[:, :, None]
    raw = (key + mu).bfloat16()
    avg = raw.float().mean(dim=2, keepdim=True).bfloat16()
    key = raw - avg                                                          # bf16 arithmetic, as the reference's fill
    value = torch.randn((B, Hkv, n, d), generator=g).bfloat16()
    win_k = (torch.randn((B, Hkv, W, d), generator=g, dtype=torch.float64) + mu).bfloat16() - avg
    win_v = torch.randn((B, Hkv, W, d), generator=g).bfloat16()
    k_new = torch.randn((B, T, Hkv, d), generator=g, dtype=torch.float64) + mu.reshape(B, 1, Hkv, d)
    v_new = torch.randn((B, T, Hkv, d), generator=g).bfloat16()
    if regime == "R4":
        q = q * 16.0
    q = q.bfloat16()
    if regime == "R5":   # stored keys that are exact power-of-two multiples of a query whose bf16 norm rounds down
        q0 = q[:, 0]
        for b in range(B):
            for h in range(Hq):
                qn32 = q0[b, h].float().norm()
                for j, sc in enumerate((1.0, 2.0, 0.5)):
                    kk = (q0[b, h].float() * sc).bfloat16()
                    if float(kk.norm().float()) < float(qn32) * sc:   # the stored bf16 norm rounds down: cs > 1 in fp32
                        key[b, h // G, (h * 7 + 101 * j) % n] = kk
    c = dict(B=B, C=B, Hq=Hq, Hkv=Hkv, G=G, n=n, K=K, L=L, hf=hf, q=q, slot_of=list(range(B)), vis=None,
             slots=[dict(value=value[b], avg=avg.reshape(B, Hkv, d)[b]) for b in range(B)], win_k=list(win_k),
             win_v=list(win_v), k_new=k_new.bfloat16(), v_new=v_new, regime=regime)
    # norm of the bf16 keys, bf16-rounded (reference)
    _set_stores(c, key, key.norm(p=2, dim=-1).float(), synth.hash_keys(key, hf, K, L))
    _tune_case(c, regime, u, place, parents)
    return c


def _tune_case(c, regime, u, place, parents):
    B, T, Hq, G = c["B"], c["q"].shape[1], c["Hq"], c["G"]
    if regime in ("R2", "R3"):
        # sink rows (and the new tokens) along the group direction; R2: strong enough that the window holds >= 90 % of the mass
        sets = sample_sets(c, cpu_codes(c))
        sigma = 2.0
        if regime == "R2":
            need = 0.0
            for b in range(B):
                for t in range(T):
                    for h in range(Hq):
                        s, off, sw, _ = _terms(c, sets, b, t, h)
                        rest = torch.logsumexp(torch.cat([s + off, sw[NS:]]), 0)
                        a = float(c["q"][b, t, h].double() @ u[b, h // G])          # sink score per unit of sigma
                        need = max(need, (float(rest) + math.log(9 * 4) + 1.0 - math.log(NS)) / a)
            sigma = need
        sink = (sigma * RD * u).bfloat16()                                          # (B, Hkv, d)
        for b in range(B):
            c["win_k"][b][:, :NS] = sink[b][:, None]
        avg = torch.stack([avg_of(c, b) for b in range(B)])
        c["k_new"] = (c["k_new"].double() * 0.25 + (sink.double() + avg.double())[:, None]).bfloat16()
    if regime == "R3":
        # per query a scale lambda (bisection) for a window share of 0.35 / 0.65 alternately
        sets = sample_sets(c, cpu_codes(c))
        q = c["q"].double().clone()
        for b in range(B):
            for t in range(T):
                for h in range(Hq):
                    target = 0.35 if h % 2 == 0 else 0.65
                    new = (c["k_new"][b, visible(parents, b, t) + [t], h // G] - avg_of(c, b)[h // G])
                    s, off, sw, _ = _terms(c, sets, b, t, h, win_extra=new)
                    lo, hi = -12.0, 12.0
                    for _ in range(60):
                        lam = 2.0 ** ((lo + hi) / 2)
                        lw, ls = torch.logsumexp(lam * sw, 0), torch.logsumexp(lam * s + off, 0)
                        if float(torch.sigmoid(lw - ls)) < target:
                            lo = (lo + hi) / 2
                        else:
                            hi = (lo + hi) / 2
                    q[b, t, h] *= 2.0 ** ((lo + hi) / 2)
        c["q"] = q.bfloat16()
    if regime == "R4":
        # one dominant key along the group direction, scaled so that it takes about half the mass of the median query
        pos = 0 if place == "first" else c["n"] - 1
        unit_key = (RD * u).bfloat16()
        for b in range(B):
            c["slots"][b]["key"][:, pos] = unit_key[b]
        _rehash(c)
        sets = sample_sets(c, cpu_codes(c))
        deltas = []
        for b, t, h in _each_head(c):
            s, off, sw, idx = _terms(c, sets, b, t, h)
            if not bool((idx == pos).any()):
                continue
            mine = idx == pos
            rest = torch.logsumexp(torch.cat([(s + off)[~mine], sw]), 0)
            deltas.append((float(rest - off[mine][0]) / float(s[mine][0])))
        assert len(deltas) * 2 >= B * T * Hq, "the dominant key is not sampled for most queries"
        delta = max(sorted(deltas)[len(deltas) // 2], 2.0 ** -6)
        for b in range(B):
            c["slots"][b]["key"][:, pos] = (unit_key[b].double() * delta).bfloat16()
        _rehash(c)
        c["dominant"] = pos


def self_check(c, name, o, run):
    """The regime's named perturbation of the restatement must move the output by >= 10x the bar."""
    moved = rel_rows(run(SELF_CHECK[name]), o)
    assert moved >= 10 * BAR, f"{name}: inputs are insensitive, '{SELF_CHECK[name]}' moves the output by {moved:.2e} only"
    return moved


def check_case(c, parents=None):
    """The generator's self-checks (fp64, CPU codes, no GPU): the regime's property holds and its perturbation is visible."""
    regime = c["regime"]
    codes = cpu_codes(c)
    sets = sample_sets(c, codes)
    o, lse_s, share = restate(c, codes, parents=parents, sets=sets)
    assert torch.isfinite(o).all()
    run = lambda v: restate(c, codes, v, parents, sets=sets)[0]   # noqa: E731
    if regime == "R2":
        assert float(share.min()) >= 0.9, f"R2: window share {float(share.min()):.3f} < 0.9"
    if regime == "R3":
        assert 0.3 <= float(share.min()) and float(share.max()) <= 0.7, f"R3: window share in [{share.min():.3f}, {share.max():.3f}]"
    if regime == "R4":
        span = []
        for b, t, h in _each_head(c):
            s, off, sw, _ = _terms(c, sets, b, t, h)
            z = torch.cat([s + off, sw])
            span.append(float(z.max() - z.min()))
        assert min(span) >= 40.0, f"R4: scores span {min(span):.1f} nats only"
    if regime == "R5":
        hit = 0
        for b in range(c["B"]):
            st = c["slots"][b]
            for h in range(c["Hq"]):
                idx = sets[b][0][h]
                qh = c["q"][b, 0, h]
                cs = (st["key"][h // c["G"], idx].float() @ qh.float()) / (qh.float().norm() * st["kn"][h // c["G"], idx])
                hit += int((cs > 1.0).sum())
        assert hit > 0, "R5: no sampled key has an fp32 cosine past 1"
    if regime in SELF_CHECK:
        self_check(c, regime, o, run)
    return o


# ---- dense layers, one prompt per request ----------------------------------------------------------------------------------
def make_dense(regime, B, Hq, Hkv, P, T, seed, place="last", one_prompt=False, dev="cpu"):
    """Dense-layer inputs: prompt rows dk/dv (B, P, Hkv, d), q (B, T, Hq, d), step rows k/v (B, T, Hkv, d), the group
    directions u (B, Hkv, d), drawn on dev.
    R2: the first NS prompt rows and the step's keys lie along the group direction (sigma sqrt(d) u) and hold >= 90 % of the
    mass; R4: queries x 16 and one dominant row at the first / last prompt row (place="new": the step's last key).
    one_prompt: every request has the same prompt (and query direction), as the requests bound to one context slot."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *s: torch.randn(s, generator=g, device=dev, dtype=torch.float64)   # noqa: E731
    G = Hq // Hkv
    u = unit(rnd, 1 if one_prompt else B, Hkv).expand(B, Hkv, d)
    q = 0.5 * rnd(B, T, Hq, d) + RD * u.repeat_interleave(G, 1)[:, None]
    dk = rnd(1 if one_prompt else B, P, Hkv, d).expand(B, P, Hkv, d).clone()
    dv = torch.randn((1 if one_prompt else B, P, Hkv, d), generator=g, device=dev).bfloat16().expand(B, P, Hkv, d).clone()
    k = rnd(B, T, Hkv, d)
    v = torch.randn((B, T, Hkv, d), generator=g, device=dev).bfloat16()
    c = dict(B=B, Hq=Hq, Hkv=Hkv, G=G, P=P, regime=regime, place=place, u=u)
    if regime == "R2":
        qq = q.bfloat16().double()
        a = torch.einsum("bthd,bhd->bth", qq, u.repeat_interleave(G, 1)).min()
        rest = math.log(P + T) + 8.0                       # every other score is below 8 nats for these queries
        sigma = (rest + math.log(9 * 2)) / float(a)
        ns = min(NS, P)
        dk[:, :ns] = sigma * RD * u[:, None]
        k = 0.25 * k + sigma * RD * u[:, None]
        c["sigma"] = sigma
    else:
        q = q * 16.0
        qq = q.bfloat16().double()
        pos = {"first": 0, "last": P - 1, "new": None}[place]
        rows = torch.cat([dk, k], dim=1)
        s = torch.einsum("btkgd,bnkd->btkgn", qq.reshape(B, T, Hkv, G, d), rows) / RD
        a = torch.einsum("btkgd,bkd->btkg", qq.reshape(B, T, Hkv, G, d), u)      # score of the row rd * u per unit of delta
        delta = float(((torch.logsumexp(s, -1) + 2.0) / a).median())               # ~90 % of the mass for the median query
        dom = delta * RD * u
        if pos is None:
            k[:, -1] = dom
        else:
            dk[:, pos] = dom
    c.update(q=q.bfloat16(), dk=dk.bfloat16(), dv=dv, k=k.bfloat16(), v=v)
    return c


def restate_dense(c, parents=None, variant=None):
    """fp64 output (B, T, Hq, d) of a dense step: prompt rows + the visible step rows (causal or ancestors) + the token.
    variant: drop_newest, skip_rescale, tree_as_chain (the ancestor mask read as a chain) or None."""
    B, T, Hq, G = c["B"], c["q"].shape[1], c["Hq"], c["G"]
    o = torch.zeros((B, T, Hq, d), dtype=torch.float64, device=c["q"].device)
    for b in range(B):
        for t in range(T):
            rows = visible(None if variant == "tree_as_chain" else parents, b, t) + [t]
            kk = torch.cat([c["dk"][b], c["k"][b, rows]])
            vv = torch.cat([c["dv"][b], c["v"][b, rows]])
            if variant == "drop_newest":
                kk, vv = kk[:-1], vv[:-1]
            if variant == "skip_rescale" and c.get("place") == "first":   # (order-free sum: visit the dominant row last)
                kk, vv = kk.flip(0), vv.flip(0)
            for h in range(Hq):
                z = (kk[:, h // G].double() @ c["q"][b, t, h].double()) / RD
                if variant == "skip_rescale":   # row-granular, so that small P still has a rescale to skip
                    o[b, t, h], _ = softmax_state(z, vv[:, h // G], True, tile=1)
                else:
                    o[b, t, h], _ = softmax_state(z, vv[:, h // G])
    return o


def dense_moves(c, parents=None, extra=()):
    """The dense generator's self-check: the regime's perturbation (R2 drop_newest, R4 skip_rescale) and the opt-in ones of
    extra must each move the fp64 output by >= 10x the bar.  Returns (output, {perturbation: how far it moves the output})."""
    o = restate_dense(c, parents)
    moved = {}
    for variant in ("drop_newest" if c["regime"] == "R2" else "skip_rescale",) + tuple(extra):
        moved[variant] = rel_rows(restate_dense(c, parents, variant), o)
        assert moved[variant] >= 10 * BAR, f"dense {c['regime']}: '{variant}' moves the output by {moved[variant]:.2e} only"
    return o, moved


def check_dense(c, parents=None):
    return dense_moves(c, parents)[0]


# ------------------------------------------------------------------------------------------------
# the steps after an accept or a rewind
# ------------------------------------------------------------------------------------------------
ACCEPT_VARIANTS = ("node_order", "path_dropped", "step_kept")


def committed_as(variant, keep, T):
    """What a wrong accept or rewind of a T-node step commits instead of keep (per request, the nodes in order): node_order --
    nodes 0 .. count - 1 (the path's length, not its nodes); path_dropped -- nothing; step_kept -- every node (the accept or
    rewind ignored)."""
    return {"node_order": [list(range(len(k))) for k in keep], "path_dropped": [[] for _ in keep],
            "step_kept": [list(range(T)) for _ in keep]}[variant]


def next_case(c, keep, T, seed):
    """The sparse case of the step after c's.  Request b's step committed c's nodes keep[b], in that order (an accepted root path,
    the first T' - r nodes after rewind(r), or none), so its window gains their rows -- keys centred as the append centres them.
    Then a step of T new tokens drawn as make_batch draws R2's: queries along the slot's group direction, keys on its sink rows,
    so that the window, committed rows included, holds the mass.  The draws depend on the seed only, not on keep."""
    assert c["regime"] == "R2", "next_case draws R2 steps"
    dev = c["q"].device
    g = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *s: torch.randn(s, generator=g, device=dev, dtype=torch.float64)   # noqa: E731
    B, Hq, Hkv, G = c["B"], c["Hq"], c["Hkv"], c["G"]
    win_k, win_v = [], []
    for b in range(B):
        rows = torch.tensor(keep[b], dtype=torch.long, device=dev)
        win_k.append(torch.cat([c["win_k"][b], centred(c["k_new"][b, rows], avg_of(c, b)).transpose(0, 1)], dim=1))
        win_v.append(torch.cat([c["win_v"][b], c["v_new"][b, rows].transpose(0, 1)], dim=1))
    U = torch.stack([c["slots"][s]["u"] for s in c["slot_of"]])
    sink = torch.stack([c["win_k"][b][:, 0].double() + avg_of(c, b).double() for b in range(B)])   # (B, Hkv, d) uncentred
    q = rnd(B, T, Hq, d) + RD * U.repeat_interleave(G, 1)[:, None]
    k_new = 0.25 * rnd(B, T, Hkv, d) + sink[:, None]
    v_new = torch.randn((B, T, Hkv, d), generator=g, device=dev).bfloat16()
    return dict(c, q=q.bfloat16(), k_new=k_new.bfloat16(), v_new=v_new, win_k=win_k, win_v=win_v)


def next_dense(c, keep, T, seed):
    """The dense case of the step after c's: c's nodes keep[b] (as many for every request) follow request b's prompt rows, in
    that order, then a step of T new tokens drawn as make_dense draws R2's.  The draws depend on the seed only."""
    assert c["regime"] == "R2", "next_dense draws R2 steps"
    assert len({len(k) for k in keep}) == 1, "every request commits as many rows"
    dev = c["q"].device
    g = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *s: torch.randn(s, generator=g, device=dev, dtype=torch.float64)   # noqa: E731
    B, Hq, Hkv, G, u = c["B"], c["Hq"], c["Hkv"], c["G"], c["u"]
    idx = [torch.tensor(k, dtype=torch.long, device=dev) for k in keep]
    dk = torch.cat([c["dk"], torch.stack([c["k"][b, idx[b]] for b in range(B)])], dim=1)
    dv = torch.cat([c["dv"], torch.stack([c["v"][b, idx[b]] for b in range(B)])], dim=1)
    q = 0.5 * rnd(B, T, Hq, d) + RD * u.repeat_interleave(G, 1)[:, None]
    k = 0.25 * rnd(B, T, Hkv, d) + c["sigma"] * RD * u[:, None]
    v = torch.randn((B, T, Hkv, d), generator=g, device=dev).bfloat16()
    return dict(c, P=dk.shape[1], q=q.bfloat16(), dk=dk, dv=dv, k=k.bfloat16(), v=v)


def after_steps(c, keep, steps, seed, nxt=next_case):
    """The cases of the steps after c's when c's step commits keep and each following step, of steps[i] tokens, commits all of
    its tokens."""
    out, cur = [], c
    for i, T in enumerate(steps):
        cur = nxt(cur, keep, T, seed + i)
        out.append(cur)
        keep = [list(range(T))] * c["B"]
    return out


def _accept_moves(c, keep, steps, seed, nxt, restate_fn, moved):
    """Every accept variant that commits other rows than keep must move the restated output of every following step by >= 10x
    the bar; moved[variant] = its smallest move."""
    refs = [restate_fn(x) for x in after_steps(c, keep, steps, seed, nxt)]
    for variant in ACCEPT_VARIANTS:
        alt = committed_as(variant, keep, c["q"].shape[1])
        if alt == keep:
            continue
        moved[variant] = min(rel_rows(restate_fn(x), o) for x, o in zip(after_steps(c, alt, steps, seed, nxt), refs))
        assert moved[variant] >= 10 * BAR, f"inputs are insensitive: '{variant}' moves a following step by {moved[variant]:.2e} only"
    return moved


def check_after(c, keep, steps, seed):
    """The sparse steps after c's (after_steps), each self-checked by check_inputs, and the accept variants (_accept_moves).
    Returns (cases, {perturbation: smallest move over the steps})."""
    cases = after_steps(c, keep, steps, seed)
    moved = {}
    for x in cases:
        for k, v in check_inputs(x).items():
            moved[k] = min(v, moved.get(k, v))

    def restate_fn(x):   # (the draws, hence the codes, are the same whichever rows were committed)
        codes = query_codes(x["q"], x["hf"], x["K"], x["L"])[0]
        return restate(x, codes)[0]
    return cases, _accept_moves(c, keep, steps, seed, next_case, restate_fn, moved)


def check_dense_after(c, keep, steps, seed):
    """The dense steps after c's (after_steps with next_dense), each self-checked by dense_moves, and the accept variants.
    Returns (cases, {perturbation: smallest move over the steps})."""
    cases = after_steps(c, keep, steps, seed, next_dense)
    moved = {}
    for x in cases:
        for k, v in dense_moves(x)[1].items():
            moved[k] = min(v, moved.get(k, v))
    return cases, _accept_moves(c, keep, steps, seed, next_dense, restate_dense, moved)


# ------------------------------------------------------------------------------------------------
# make_batch: B requests on C slots at the measured shapes
# ------------------------------------------------------------------------------------------------
def make_batch(regime, B, C=1, n=N_C2, T=1, lens=LENS, place="key", seed=0, dev=DEV, Hq=HQ, Hkv=HKV, K=KK, L=LL,
               parents=None, dominant=None, base=None):
    """Sparse-layer inputs of one regime for B requests bound to C slots (request b on slot b % C).  Per slot: key / value
    (Hkv, n, d) centred store, kn, avg (Hkv, d), kcodes (fp64), the group directions u.  Per request: its window win_k / win_v
    (Hkv, w_b, d) centred, w_b = lens[b % len(lens)] - T filled rows; q (B, T, Hq, d), k_new / v_new (B, T, Hkv, d) as the model
    produces them (uncentred).  R4: place = "key" (stored key `dominant`, default the last, dominates) or "win" (every request's
    last window row).  base: an earlier case of the same regime, C, n and heads whose hash functions and stores (copied, without
    their R4 dominant key: generate it with place = "win") to reuse instead of drawing new ones; the seed draws the rest."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *s: torch.randn(s, generator=g, device=dev, dtype=torch.float64)   # noqa: E731
    G = Hq // Hkv
    hf = synth.make_hash_func(d, K, L, seed=seed + 1).to(dev) if base is None else base["hf"]
    slots = [] if base is None else [dict(st, key=st["key"].clone(), kn=st["kn"].clone(), kcodes=st["kcodes"].clone())
                                     for st in base["slots"]]
    for _ in range(C if base is None else 0):
        u = unit(rnd, Hkv)
        mu = torch.zeros((Hkv, 1, d), dtype=torch.float64, device=dev)
        if regime == "R1":   # |mu| ~ 4 |noise|, partly along the queries
            mu = 4.0 * (0.8 * rnd(Hkv, 1, d) + 0.6 * RD * u[:, None])
        key = rnd(Hkv, n, d)
        if regime != "R4":   # a share of the keys clusters around the group direction, so that K10 L150 samples some of them
            pull = (torch.rand((Hkv, n, 1), generator=g, device=dev) < 0.125) * torch.rand((Hkv, n, 1), generator=g, device=dev) * 1.2
            key = key + pull * RD * u[:, None]
        raw = (key + mu).bfloat16()
        del key
        avg = raw.float().mean(dim=1, keepdim=True).bfloat16()
        key = raw - avg
        slots.append(dict(u=u, mu=mu, key=key, value=torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16(),
                          avg=avg.reshape(Hkv, d), kn=key.norm(p=2, dim=-1).float(), kcodes=key_codes(key, hf, K, L)))
    slot_of = [b % C for b in range(B)]
    U = torch.stack([slots[s]["u"] for s in slot_of])
    MU = torch.stack([slots[s]["mu"] for s in slot_of])
    q = (0.5 if regime == "R4" else 1.0) * rnd(B, T, Hq, d) + RD * U.repeat_interleave(G, 1)[:, None]
    if regime == "R4":
        q = q * 16.0
    w = [lens[b % len(lens)] - T for b in range(B)]
    # half the window rows lean towards the group direction, so that the window carries mass in every regime and a request
    # reading another request's window is visible
    win_k = []
    for b in range(B):
        pull = (torch.rand((Hkv, w[b], 1), generator=g, device=dev) < 0.5) * torch.rand((Hkv, w[b], 1), generator=g, device=dev)
        win_k.append((rnd(Hkv, w[b], d) + pull * RD * U[b][:, None] + MU[b]).bfloat16() - slots[slot_of[b]]["avg"][:, None])
    win_v = [torch.randn((Hkv, w[b], d), generator=g, device=dev).bfloat16() for b in range(B)]
    c = dict(B=B, C=C, Hq=Hq, Hkv=Hkv, G=G, K=K, L=L, n=n, hf=hf, slots=slots, slot_of=slot_of, regime=regime, place=place,
             q=q.bfloat16(), win_k=win_k, win_v=win_v, k_new=(rnd(B, T, Hkv, d) + MU.reshape(B, 1, Hkv, d)).bfloat16(),
             v_new=torch.randn((B, T, Hkv, d), generator=g, device=dev).bfloat16(), vis=None)
    _tune_batch(c, regime, place, parents, c["n"] - 1 if dominant is None else dominant)
    return c


def _tune_batch(c, regime, place, parents, pos):
    G = c["G"]
    if regime == "R2":
        # sink rows (and the new tokens) along the group direction, strong enough that the window holds >= 90 % of the mass
        sets = sample_sets(c, query_codes(c["q"], c["hf"], c["K"], c["L"])[0])
        need = 0.0
        for b, t, h in _each_head(c):
            s, off, sw, _ = _terms(c, sets, b, t, h)
            rest = torch.logsumexp(torch.cat([s + off, sw[NS:]]), 0)
            a = float(c["q"][b, t, h].double() @ c["slots"][c["slot_of"][b]]["u"][h // G])
            need = max(need, (float(rest) + math.log(9 * 4) + 1.0 - math.log(NS)) / a)
        for b in range(c["B"]):
            st = c["slots"][c["slot_of"][b]]
            sink = (need * RD * st["u"]).bfloat16()
            c["win_k"][b][:, :NS] = sink[:, None]
            c["k_new"][b] = (c["k_new"][b].double() * 0.25 + (sink.double() + st["avg"].double())[None]).bfloat16()
    if regime == "R4" and place == "key":
        # stored key pos of every slot (by default the last: last key segment, last tile of its CTA's sample) along the group
        # direction, scaled so that it takes about half the mass of the median query that samples it
        for st in c["slots"]:
            st["key"][:, pos] = (RD * st["u"]).bfloat16()
            st["kn"][:, pos] = st["key"][:, pos].norm(p=2, dim=-1).float()
            st["kcodes"][:, :, pos:pos + 1] = key_codes(st["key"][:, pos:pos + 1], c["hf"], c["K"], c["L"])
        sets = sample_sets(c, query_codes(c["q"], c["hf"], c["K"], c["L"])[0])
        deltas = [[] for _ in c["slots"]]
        for b, t, h in _each_head(c):
            s, off, sw, idx = _terms(c, sets, b, t, h)
            mine = idx == pos
            if not bool(mine.any()):
                continue
            rest = torch.logsumexp(torch.cat([(s + off)[~mine], sw]), 0)
            deltas[c["slot_of"][b]].append(float(rest - off[mine][0]) / float(s[mine][0]))
        assert sum(map(len, deltas)) * 2 >= len(_each_head(c)), "the dominant key is not sampled for most queries"
        for st, ds in zip(c["slots"], deltas):
            delta = max(sorted(ds)[len(ds) // 2], 2.0 ** -6)
            st["key"][:, pos] = (RD * st["u"] * delta).bfloat16()
            st["kn"][:, pos] = st["key"][:, pos].norm(p=2, dim=-1).float()
            st["kcodes"][:, :, pos:pos + 1] = key_codes(st["key"][:, pos:pos + 1], c["hf"], c["K"], c["L"])
        c["dominant"] = pos
    if regime == "R4" and place == "win":
        # every request's last filled window row (in the window's last tile) dominates, about half the median query's mass
        sets = sample_sets(c, query_codes(c["q"], c["hf"], c["K"], c["L"])[0])
        for b in range(c["B"]):
            c["win_k"][b][:, -1] = (RD * c["slots"][c["slot_of"][b]]["u"]).bfloat16()
        deltas = []
        for b, t, h in _each_head(c):
            s, off, sw, _ = _terms(c, sets, b, t, h)
            rest = torch.logsumexp(torch.cat([s + off, sw[:-1]]), 0)
            deltas.append(float(rest) / float(sw[-1]))
        delta = max(sorted(deltas)[len(deltas) // 2], 2.0 ** -6)
        for b in range(c["B"]):
            c["win_k"][b][:, -1] = (RD * c["slots"][c["slot_of"][b]]["u"] * delta).bfloat16()


def pick(x, c, heads):
    """The rows of the chosen heads of a (B, T, Hq, d) or (B*T*Hq, d) tensor, as (rows, d)."""
    B, Hq = c["B"], c["Hq"]
    x = x.reshape(B, -1, Hq, d).transpose(1, 2)
    return x[head_mask(c, heads).to(x.device)].reshape(-1, d)


def perturbations(c):
    """The named perturbations the case's inputs must make visible."""
    names = [SELF_CHECK[c["regime"]]]
    if c["B"] > 1 and len({w.shape[1] for w in c["win_k"]}) > 1:
        names.append("window_of_request_0")
    if c["C"] >= 2 and (c["regime"] == "R1" or c["place"] == "key" and c["regime"] == "R4"):   # the store carries mass
        names.append("wrong_document")
    if c["regime"] == "R1":   # the sampled half carries nearly all the mass of every head
        names.append("drop_sampled")
    return names


def check_inputs(c, parents=None, heads=None, extra=()):
    """The generator's self-checks on fp64 query codes, before any library call: the regime's property holds and every named
    perturbation (those of the case, then the opt-in ones of extra, e.g. tree_as_chain) moves the restated output by >= 10x the
    bar.  Returns {perturbation: how far it moves the output}."""
    codes = query_codes(c["q"], c["hf"], c["K"], c["L"])[0]
    sets = sample_sets(c, codes)
    o, _, share = restate(c, codes, parents=parents, heads=heads, sets=sets)
    assert bool(torch.isfinite(o).all())
    hm = head_mask(c, heads)[:, None].expand(share.shape)
    if c["regime"] == "R2":
        assert float(share[hm].min()) >= 0.9, f"R2: window share {float(share[hm].min()):.3f} < 0.9"
    if c["regime"] == "R4":
        span = []
        for b, t, h in _each_head(c):
            if hm[b, t, h]:
                s, off, sw, _ = _terms(c, sets, b, t, h)
                z = torch.cat([s + off, sw])
                span.append(float(z.max() - z.min()))
        assert min(span) >= 40.0, f"R4: scores span {min(span):.1f} nats only"
    moved = {}
    for name in perturbations(c) + list(extra):
        a = pick(restate(c, codes, name, parents, heads, sets=None if name == "wrong_document" else sets)[0], c, heads)
        b = pick(o, c, heads)
        per_head = (a - b).abs().amax(-1) / b.abs().amax(-1).clamp_min(1e-30)
        moved[name] = float(per_head.min() if name in EVERY_HEAD else per_head.max())
        assert moved[name] >= 10 * BAR, f"inputs are insensitive: '{name}' moves the output by {moved[name]:.2e} only"
    return moved


# ---- dense layers in shared-prefix mode ------------------------------------------------------------------------------------
def make_dense_slots(regime, B, P, T, seed, dev=DEV, Hq=HQ, Hkv=HKV, pre=((1, 3, 0, 2), (3, 2, 0, 1))):
    """One prompt dk / dv (P, Hkv, d) for every request, then two earlier steps of 4 tokens of which request b kept
    4 - pre[i][b % 4] rows (its tail), then the step: q (B, T, Hq, d), k / v (B, T, Hkv, d).
    R2: the first NS prompt rows, the tails and the step's keys along the group direction hold >= 90 % of the mass;
    R4: queries x 16 and one dominant row, the prompt's last, with tail rows a few nats below it.  Either way the tails carry
    much of the mass, so that a request reading another's tail is visible."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *s: torch.randn(s, generator=g, device=dev, dtype=torch.float64)   # noqa: E731
    G = Hq // Hkv
    u = unit(rnd, Hkv)
    q = 0.5 * rnd(B, T, Hq, d) + RD * u.repeat_interleave(G, 0)
    dk = rnd(P, Hkv, d)
    dv = torch.randn((P, Hkv, d), generator=g, device=dev).bfloat16()
    pre_k = [rnd(B, 4, Hkv, d) for _ in pre]
    pre_v = [torch.randn((B, 4, Hkv, d), generator=g, device=dev).bfloat16() for _ in pre]
    pre_q = [rnd(B, 4, Hq, d).bfloat16() for _ in pre]
    drops = [[dr[b % len(dr)] for b in range(B)] for dr in pre]
    k = rnd(B, T, Hkv, d)
    v = torch.randn((B, T, Hkv, d), generator=g, device=dev).bfloat16()
    if regime == "R2":
        a = float(torch.einsum("bthd,hd->bth", q.bfloat16().double(), u.repeat_interleave(G, 0)).min())
        sigma = (math.log(P + 8 + T) + 8.0 + math.log(9 * 2)) / a   # every other score is below 8 nats for these queries
        dk[:NS] = sigma * RD * u
        k = 0.25 * k + sigma * RD * u
        pre_k = [0.25 * pk + sigma * RD * u for pk in pre_k]
    else:
        q = q * 16.0
        qq = q.bfloat16().double().reshape(B, T, Hkv, G, d)
        lse = torch.stack([torch.logsumexp(torch.einsum("tkgd,nkd->tkgn", qq[b], dk) / RD, -1) for b in range(B)])
        a = torch.einsum("btkgd,kd->btkg", qq, u)
        delta = float(((lse + 2.0) / a).median())
        dk[P - 1] = delta * RD * u
        pre_k = [0.25 * pk + 0.97 * delta * RD * u for pk in pre_k]
    pre_k = [pk.bfloat16() for pk in pre_k]
    tails = [(torch.cat([pk[b, :4 - dr[b]] for pk, dr in zip(pre_k, drops)]),
              torch.cat([pv[b, :4 - dr[b]] for pv, dr in zip(pre_v, drops)])) for b in range(B)]
    return dict(B=B, Hq=Hq, Hkv=Hkv, G=G, P=P, regime=regime, q=q.bfloat16(), dk=dk.bfloat16(), dv=dv, k=k.bfloat16(), v=v,
                pre=list(zip(pre_q, pre_k, pre_v, drops)), tails=tails)


def restate_dense_slots(c, variant=None):
    """fp64 output (B, T, Hq, d) of the dense step: prompt + request b's tail + the step's rows before token t + token t."""
    B, T, Hq, G = c["B"], c["q"].shape[1], c["Hq"], c["G"]
    o = torch.zeros((B, T, Hq, d), dtype=torch.float64, device=c["q"].device)
    for b in range(B):
        tk, tv = c["tails"][0 if variant == "tail_of_request_0" else b]
        for t in range(T):
            kk = torch.cat([c["dk"], tk, c["k"][b, :t + 1]])
            vv = torch.cat([c["dv"], tv, c["v"][b, :t + 1]])
            if variant == "drop_newest":
                kk, vv = kk[:-1], vv[:-1]
            for g in range(c["Hkv"]):
                z = (kk[:, g].double() @ c["q"][b, t, g * G:(g + 1) * G].double().t()) / RD      # (rows, G)
                if variant == "skip_rescale":   # row-granular, as restate_dense
                    for j in range(G):
                        o[b, t, g * G + j], _ = softmax_state(z[:, j], vv[:, g], True, tile=1)
                else:
                    o[b, t, g * G:(g + 1) * G] = torch.softmax(z, 0).t() @ vv[:, g].double()
    return o


def check_dense_inputs(c):
    o = restate_dense_slots(c)
    moved = {}
    for name in ("drop_newest" if c["regime"] == "R2" else "skip_rescale", "tail_of_request_0"):
        moved[name] = rel_rows(restate_dense_slots(c, name), o)
        assert moved[name] >= 10 * BAR, f"dense {c['regime']}: '{name}' moves the output by {moved[name]:.2e} only"
    return o, moved


# ------------------------------------------------------------------------------------------------
# GPU side
# ------------------------------------------------------------------------------------------------
def seed_of(*key):
    return zlib.crc32(repr(key).encode()) % 10000


def fill_case(ctx, c):
    """Fill ctx from case c: each slot through its first request, the other requests forked onto it (or, with one slot per
    request in ctx, filled themselves), then every request's own window."""
    put = lambda x: x.to(DEV).contiguous()   # noqa: E731
    for b in range(c["B"]):
        if b < c["C"] or ctx.num_contexts >= c["B"]:
            st = c["slots"][c["slot_of"][b]]
            ctx.attn_fill(1, b, put(st["key"]), put(st["value"]), put(st["kn"]))
            ctx.lsh_build(1, b, put(st["kcodes"]))
        else:
            ctx.fork(c["slot_of"][b], b)
    for b in range(c["B"]):
        ctx.window_fill(1, b, put(avg_of(c, b)), put(c["win_k"][b]), put(c["win_v"][b]))
    return ctx


def batch_ctx(c, C=1, M=M_C2, gen=GEN, kreg=0, save_mask=1, t_max=1, shared_spill=False):
    """A context over case c's slots (fill_case)."""
    ctx = two_layer_context(c["K"], c["L"], c["Hq"], c["Hkv"], c["B"], M, gen, c["hf"],
                            dict(decode_impl=1, fused_kreg=kreg, save_mask=save_mask, out_f32=1), max_query_tokens=t_max,
                            num_contexts=C, shared_spill=shared_spill)
    return fill_case(ctx, c)


def step(ctx, c, parents=None, lists=True):
    """One step of c's T tokens; readouts shaped (B, T, Hq, ...) on the device."""
    B, T, Hq = c["q"].shape[:3]
    if T == 1:
        ctx.plan()
        out = ctx.decode(1, c["q"][:, 0].contiguous(), c["k_new"][:, 0].contiguous(), c["v_new"][:, 0].contiguous())
    else:
        ctx.plan(T, parents=None if parents is None else torch.tensor(parents, dtype=torch.int32, device=DEV))
        out = ctx.decode_tokens(1, T, c["q"].contiguous(), c["k_new"].contiguous(), c["v_new"].contiguous())
    nnz, res = ctx.last_probe(want_results=lists)
    r = dict(out=out.reshape(B, T, Hq, d), o32=ctx.last_out_f32().reshape(B, T, Hq, d), nnz=nnz.reshape(B, T, Hq),
             fused=ctx.get_info("last_decode_fused"))
    if lists:
        r.update(res=res.reshape(B, T, Hq, -1), codes=ctx.last_codes().reshape(B, T, Hq, -1))
    return r


def twin_lists(r, rt, label):
    """Codes and lists of a save_mask = 0 step r from the same step rt of a save_mask = 1 twin filled identically, which must
    have run the fused kernel and sampled the same counts."""
    assert rt["fused"] == 1, f"{label}: the twin did not run the fused kernel"
    assert torch.equal(r["nnz"], rt["nnz"]), f"{label}: save_mask = 0 sampled other counts than its twin"
    r.update(res=rt["res"], codes=rt["codes"])
    return r


def twin_step(make_ctx, c, label, parents=None, fused=True, hook=None):
    """One step of case c on the context make_ctx(save_mask) returns.  Fused steps run as the measured lines run them, with
    save_mask = 0 (the CTAs list their selection in the carved extra row buffers), and take their codes and lists from a
    save_mask = 1 twin (twin_lists); the three-launch path always writes its lists.  hook(ctx, r) sees the context before it is
    released, which happens before the twin is made."""
    save_mask = 0 if fused else 1
    ctx = make_ctx(save_mask)
    r = step(ctx, c, parents, lists=bool(save_mask))
    assert r["fused"] == int(fused), f"{label}: last_decode_fused = {r['fused']}"
    if hook is not None:
        hook(ctx, r)
    del ctx
    if fused:
        tw = make_ctx(1)
        rt = step(tw, c, parents)
        del tw
        twin_lists(r, rt, label)
    return r


def check_codes_lists(c, r):
    """GPU query codes against the fp64 projection (a code may differ only where a projection is within SIMHASH_EPS of zero);
    nnz and index lists exactly the keys of the request's slot that collide in >= 2 tables.  Returns the sample sets."""
    ref, margin = query_codes(c["q"], c["hf"], c["K"], c["L"])
    bad = r["codes"] != ref
    if bool(bad.any()):
        assert float(margin[bad].max()) < SIMHASH_EPS, f"{int(bad.sum())} query codes differ beyond rounding"
    sets = sample_sets(c, r["codes"])
    B, T, Hq = r["nnz"].shape
    want = torch.tensor([[[len(sets[b][t][h]) for h in range(Hq)] for t in range(T)] for b in range(B)], dtype=torch.int32)
    assert torch.equal(r["nnz"].cpu(), want), "nnz differ from the collision counts"
    for b in range(B):
        for t in range(T):
            for h in range(Hq):
                assert torch.equal(r["res"][b, t, h, : int(want[b, t, h])].long(), sets[b][t][h]), (b, t, h)
    return sets


def check_outputs(c, r, sets, label, parents=None, heads=None):
    """fp32 output within 1e-3 of the fp64 restatement per head; bf16 output = fp32 rounded once.  Prints the worst head."""
    o = restate(c, r["codes"], parents=parents, heads=heads, sets=sets)[0]
    worst = rel_rows(pick(r["o32"], c, heads), pick(o, c, heads))
    print(f"{label}: largest relative head error {worst:.2e} ({worst / BAR:.1%} of the bar)")
    assert worst <= BAR, f"{label}: fp32 output differs from fp64 by {worst:.3e} relative (bar {BAR:g})"
    assert_rounded_half_up(r["out"], r["o32"], label)
    return worst
