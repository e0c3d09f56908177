"""Batched decode over one long context against fp64, at the shapes the shared-context, beam and long-generation lines measure
(`-m gpu`).

Those lines run Llama-3.1-8B heads (Hq 32, Hkv 8, K10 L150) over one 98 K-token context at B = 1 ... 32.  The other fp64 file
(test_gpu_numerics.py) stops at B <= 4 and n <= 70 000 with one slot per request and equal window lengths, and the B = 8 test at
this size (test_gpu_shared.py::test_c2_size_b8_one_context) compares two contexts that run the same kernels.  Here every request
of a step is checked against an fp64 restatement of ITS slot's store and ITS own window:

  * the path each measured shape runs is pinned (test_measured_shapes_path): fused at B <= 4, the three-launch path
    (simhash -> probe -> stream-K attend) at B >= 8, the fused T-token kernel in several waves for T = 4;
  * one C2-size context (n = 97 932, M = 98 304, or 131 072 with shared spill) per slot, on the device; the key codes are an
    fp64 GEMM (`key_codes`) handed to lsh_build, so the tables do not depend on the key-hash kernel;
  * ragged windows (69, 150, 324, 200 rows cycled over the requests, 324 = the full window of generation_buffer 256), windows
    of 4 000 ... 4 172 rows, two documents on two slots, 1 024 heads in one step, T = 4 chains and an 8-node tree, a step after a
    shared spill and after a fork of a request that spilled, and the dense layers in shared-prefix mode at B = 8 and 32.

Regimes (the knobs of test_gpu_numerics.py): R1 key mean, R2 sinks (the window holds >= 90 % of the mass), R4 large logits with
one dominant row, either the LAST stored key (last key segment, last sampled tile) or the last window row of every request.
Before any library call each case checks that its named perturbations of the restatement move the output by >= 10x the 1e-3
bar: the regime's own (SELF_CHECK) and, for batches, `window_of_request_0` (every request attends over request 0's window) and,
with two slots whose stores carry the mass (R1, R4 with a dominant key), `wrong_document` (request b attends over the other
slot's store); in R1, where the sampled half carries nearly all the mass, `drop_sampled` must move EVERY checked head.  Fused
steps run with save_mask = 0, as the measured lines do, and take their codes and lists from a save_mask = 1 twin.
tests/test_batch_numerics_inputs_cpu.py runs the same generator and restatement at a reduced size without a GPU.

The fp64 work runs with torch on whichever device holds the case (IEEE fp64 tensor arithmetic, none of the library's kernels).
"""
import math
import zlib

import pytest
import torch

from magicpig_b200 import synth
from tests.test_gpu_numerics import BAR, SELF_CHECK, lsh_weight, merge2, sample_scores, softmax_state, visible
from tests.test_gpu_parity import SIMHASH_EPS
from tests.test_gpu_tokens import bf16_half_up

DEV = "cuda:0"
d, NS, NL, GEN = 128, 4, 64, 256
HQ, HKV, KK, LL = 32, 8, 10, 150
N_C2, M_C2, M_LONG = 97932, 98304, 131072
LENS = (69, 150, 324, 200)            # window rows after the step, cycled over the requests (324 = NS + NL + GEN: full)
LONG_GEN = 4104                       # generation_buffer of the long-generation line's "no spill" arm: windows of up to 4 172 rows
LONG_LENS = (4000, 4172, 4100, 4050)
TREE = [-1, 0, 0, 1, 1, 2, 3, 3]
RD = math.sqrt(d)


# ------------------------------------------------------------------------------------------------
# generator: one store per context slot, every request its own window
# ------------------------------------------------------------------------------------------------
def key_codes(key: torch.Tensor, hf: torch.Tensor, K: int, L: int, chunk: int = 16384) -> torch.Tensor:
    """int16 codes (Hkv, L, n) of keys (Hkv, n, d) from the fp64 projection key @ hf, packed as synth.hash_keys."""
    Hkv, n, _ = key.shape
    pack = 2 ** torch.arange(K, device=key.device)
    hfd = hf.double().to(key.device)
    out = torch.empty((Hkv, L, n), dtype=torch.int16, device=key.device)
    for g in range(Hkv):
        for s in range(0, n, chunk):
            bits = ((key[g, s:s + chunk].double() @ hfd) > 0).reshape(-1, L, K).long()
            out[g, :, s:s + chunk] = (bits * pack).sum(-1).t().to(torch.int16)
    return out


def query_codes(q: torch.Tensor, hf: torch.Tensor, K: int, L: int):
    """int32 codes (..., L) of bf16 queries normalised as the reference (bf16 norm, bf16 quotient), fp64 projection; and per
    code the smallest |projection| of its K bits (the SIMHASH_EPS margin)."""
    nq = q / q.norm(p=2, dim=-1, keepdim=True)
    proj = (nq.double() @ hf.double().to(q.device)).reshape(*q.shape[:-1], L, K)
    codes = ((proj > 0).long() * (2 ** torch.arange(K, device=q.device))).sum(-1).int()
    return codes, proj.abs().min(dim=-1).values


def _unit(rnd, *shape):
    u = rnd(*shape, d)
    return u / u.norm(dim=-1, keepdim=True)


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
        u = _unit(rnd, Hkv)
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
    _tune(c, regime, place, parents, c["n"] - 1 if dominant is None else dominant)
    return c


def avg_of(c, b):
    return c["slots"][c["slot_of"][b]]["avg"]


def batch_sets(c, codes, wrong=False):
    """Index lists (ascending) of the keys of request b's slot (the other slot: wrong) that collide with its query codes in >= 2
    tables, restricted to the keys it sees (c["vis"], after a shared spill): codes int32 (B, T, Hq, L) -> [b][t][h]."""
    B, T, Hq = codes.shape[:3]
    G, L = c["G"], c["L"]
    out = []
    for b in range(B):
        s = (c["slot_of"][b] + 1) % c["C"] if wrong else c["slot_of"][b]
        kc = c["slots"][s]["kcodes"]
        rows = []
        for t in range(T):
            heads = []
            for g in range(c["Hkv"]):
                qc = codes[b, t, g * G:(g + 1) * G].to(kc.device, torch.int16)
                cnt = torch.zeros((G, kc.shape[-1]), dtype=torch.int64, device=kc.device)
                for l0 in range(0, L, 25):
                    cnt += (kc[g, None, l0:l0 + 25] == qc[:, l0:l0 + 25, None]).sum(dim=1)
                hit = cnt > 1
                if c["vis"] is not None and not wrong:
                    hit &= c["vis"][b][None]
                heads += [torch.nonzero(hit[j]).flatten() for j in range(G)]
            rows.append(heads)
        out.append(rows)
    return out


def _window(c, b, t, g, variant=None, parents=None):
    """Request b's window rows for token t of group g: its filled rows, the step's visible rows and the token, centred."""
    wb = 0 if variant == "window_of_request_0" else b
    new = c["k_new"][b, :, g] if variant == "uncentred" else c["k_new"][b, :, g] - avg_of(c, b)[g]
    vis = visible(parents, b, t)
    wk = torch.cat([c["win_k"][wb][g], new[vis], new[t:t + 1]])
    wv = torch.cat([c["win_v"][wb][g], c["v_new"][b, vis, g], c["v_new"][b, t:t + 1, g]])
    if variant == "drop_newest":
        wk, wv = wk[:-1], wv[:-1]
    return wk, wv


def head_mask(c, heads):
    return torch.ones((c["B"], c["Hq"]), dtype=torch.bool) if heads is None else heads


def restate_batch(c, codes, variant=None, parents=None, heads=None, sets=None):
    """fp64 output (B, T, Hq, d) of the sparse decode step of case c over each request's slot store and own window, and the
    window's share (B, T, Hq) of the merged mass.  heads: bool (B, Hq), the heads to restate (None: all)."""
    B, T, Hq = codes.shape[:3]
    G, K, L = c["G"], c["K"], c["L"]
    wrong = variant == "wrong_document"
    if sets is None:
        sets = batch_sets(c, codes, wrong)
    hm = head_mask(c, heads)
    dev = c["q"].device
    o = torch.zeros((B, T, Hq, d), dtype=torch.float64, device=dev)
    share = torch.ones((B, T, Hq), dtype=torch.float64)
    for b in range(B):
        st = c["slots"][(c["slot_of"][b] + 1) % c["C"] if wrong else c["slot_of"][b]]
        for t in range(T):
            for g in range(c["Hkv"]):
                hs = [h for h in range(g * G, (g + 1) * G) if hm[b, h]]
                if not hs:
                    continue
                wk, wv = _window(c, b, t, g, variant, parents)
                for h in hs:
                    qh, idx = c["q"][b, t, h], sets[b][t][h]
                    zs = sample_scores(qh, st["key"][g, idx], st["kn"][g, idx], K, L)
                    qw = c["q"][b, t, g * G] if variant == "window_of_head_0" else qh
                    zw = (wk.double() @ qw.double()) / RD
                    if variant == "skip_rescale":
                        o[b, t, h], _ = softmax_state(torch.cat([zw, zs]), torch.cat([wv, st["value"][g, idx]]), True)
                        continue
                    o_s, l_s = softmax_state(zs, st["value"][g, idx])
                    o_w, l_w = softmax_state(zw, wv)
                    if variant == "drop_sampled":
                        o[b, t, h] = o_w
                        continue
                    o[b, t, h] = merge2(o_w, l_w, o_s, l_s, natural=(variant == "ln_merge"))
                    share[b, t, h] = 1.0 / (1.0 + 2.0 ** (l_s - l_w)) if l_s > -math.inf else 1.0
    return o, share


def pick(x, c, heads):
    """The rows of the chosen heads of a (B, T, Hq, d) or (B*T*Hq, d) tensor, as (rows, d)."""
    B, Hq = c["B"], c["Hq"]
    x = x.reshape(B, -1, Hq, d).transpose(1, 2)
    return x[head_mask(c, heads).to(x.device)].reshape(-1, d)


def rel_heads(a, o):
    """max over heads of max|a - o| / max|o| (the bar's metric)."""
    a, o = a.double().reshape(-1, d), o.double().to(a.device).reshape(-1, d)
    return float(((a - o).abs().amax(-1) / o.abs().amax(-1).clamp_min(1e-30)).max())


def _terms(c, sets, b, t, h, parents=None):
    """Raw sampled scores s / sqrt(d), their LSH offsets -log(w + 1e-4) and the window scores (filled rows) of one head."""
    st, g = c["slots"][c["slot_of"][b]], h // c["G"]
    qh = c["q"][b, t, h].double()
    idx = sets[b][t][h]
    s = st["key"][g, idx].double() @ qh
    cs = s / (qh.norm() * st["kn"][g, idx].double())
    off = -torch.log(lsh_weight(cs, c["K"], c["L"]) + 1e-4)
    return s / RD, off, (c["win_k"][b][g].double() @ qh) / RD, idx


def _each_head(c):
    B, T, Hq = c["q"].shape[:3]
    return [(b, t, h) for b in range(B) for t in range(T) for h in range(Hq)]


def _tune(c, regime, place, parents, pos):
    G, Hkv = c["G"], c["Hkv"]
    if regime == "R2":
        # sink rows (and the new tokens) along the group direction, strong enough that the window holds >= 90 % of the mass
        sets = batch_sets(c, query_codes(c["q"], c["hf"], c["K"], c["L"])[0])
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
        sets = batch_sets(c, query_codes(c["q"], c["hf"], c["K"], c["L"])[0])
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
        sets = batch_sets(c, query_codes(c["q"], c["hf"], c["K"], c["L"])[0])
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


EVERY_HEAD = {"drop_sampled"}   # perturbations that must move every checked head, not only the most sensitive one


def check_inputs(c, parents=None, heads=None):
    """The generator's self-checks on fp64 query codes, before any library call: the regime's property holds and every named
    perturbation moves the restated output by >= 10x the bar.  Returns {perturbation: how far it moves the output}."""
    codes = query_codes(c["q"], c["hf"], c["K"], c["L"])[0]
    sets = batch_sets(c, codes)
    o, share = restate_batch(c, codes, parents=parents, heads=heads, sets=sets)
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
    for name in perturbations(c):
        a = pick(restate_batch(c, codes, name, parents, heads, sets=None if name == "wrong_document" else sets)[0], c, heads)
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
    u = _unit(rnd, Hkv)
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
                if variant == "skip_rescale":   # row-granular, as test_gpu_numerics.restate_dense
                    for j in range(G):
                        o[b, t, g * G + j], _ = softmax_state(z[:, j], vv[:, g], True, tile=1)
                else:
                    o[b, t, g * G:(g + 1) * G] = torch.softmax(z, 0).t() @ vv[:, g].double()
    return o


def check_dense_inputs(c):
    o = restate_dense_slots(c)
    moved = {}
    for name in ("drop_newest" if c["regime"] == "R2" else "skip_rescale", "tail_of_request_0"):
        moved[name] = rel_heads(restate_dense_slots(c, name), o)
        assert moved[name] >= 10 * BAR, f"dense {c['regime']}: '{name}' moves the output by {moved[name]:.2e} only"
    return o, moved


# ------------------------------------------------------------------------------------------------
# GPU side
# ------------------------------------------------------------------------------------------------
def batch_ctx(c, C=1, M=M_C2, gen=GEN, kreg=0, save_mask=1, t_max=1, shared_spill=False):
    """A context over case c's slots: each slot filled through its first request, the other requests forked onto it, then every
    request's own window."""
    from magicpig_b200.ops import Context
    ctx = Context(c["K"], c["L"], 2, c["Hq"], c["Hkv"], d, c["B"], M, NS, NL, gen, dense_layers=[0], device=DEV,
                  max_query_tokens=t_max, num_contexts=C, shared_spill=shared_spill)
    for key, val in dict(decode_impl=1, fused_kreg=kreg, save_mask=save_mask, out_f32=1).items():
        ctx.set_option(key, val)
    ctx.set_hash_func(c["hf"].contiguous())
    nslots = ctx.num_contexts
    for s in range(c["C"]):
        st = c["slots"][s]
        ctx.attn_fill(1, s, st["key"].contiguous(), st["value"].contiguous(), st["kn"].contiguous())
        ctx.lsh_build(1, s, st["kcodes"].contiguous())
    for b in range(c["C"], c["B"]):
        if nslots < c["B"]:
            ctx.fork(c["slot_of"][b], b)
        else:   # one slot per request (B = 1)
            st = c["slots"][c["slot_of"][b]]
            ctx.attn_fill(1, b, st["key"].contiguous(), st["value"].contiguous(), st["kn"].contiguous())
            ctx.lsh_build(1, b, st["kcodes"].contiguous())
    for b in range(c["B"]):
        ctx.window_fill(1, b, avg_of(c, b).contiguous(), c["win_k"][b].contiguous(), c["win_v"][b].contiguous())
    return ctx


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


def check_codes_lists(c, r):
    """GPU query codes against the fp64 projection (a code may differ only where a projection is within SIMHASH_EPS of zero);
    nnz and index lists exactly the keys of the request's slot that collide in >= 2 tables.  Returns the sample sets."""
    ref, margin = query_codes(c["q"], c["hf"], c["K"], c["L"])
    bad = r["codes"] != ref
    if bool(bad.any()):
        assert float(margin[bad].max()) < SIMHASH_EPS, f"{int(bad.sum())} query codes differ beyond rounding"
    sets = batch_sets(c, r["codes"])
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
    o, _ = restate_batch(c, r["codes"], parents=parents, heads=heads, sets=sets)
    worst = rel_heads(pick(r["o32"], c, heads), pick(o, c, heads))
    print(f"{label}: largest relative head error {worst:.2e} ({worst / BAR:.1%} of the bar)")
    assert worst <= BAR, f"{label}: fp32 output differs from fp64 by {worst:.3e} relative (bar {BAR:g})"
    assert torch.equal(r["out"].cpu().view(torch.int16).int() & 0xFFFF, bf16_half_up(r["o32"]).reshape(r["out"].shape))
    return worst


def seed_of(*key):
    return zlib.crc32(repr(key).encode()) % 10000


def skip_unless_132_sms():
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the pinned paths are those of a 132-SM H100")


# ---- 1. the path each measured shape runs --------------------------------------------------------------------------------
# (B, T, max_length, shared_spill): fused_applicable, fused_cluster_waves, last_decode_fused, tokens_cluster_waves (T > 1)
PATHS = [
    ((1, 1, M_C2, False), (1, 1, 1, None)),     # bench.py: 32 clusters of two 1024-thread CTAs
    ((2, 1, M_C2, False), (1, 1, 1, None)),
    ((4, 1, M_C2, False), (1, 1, 1, None)),     # 512-thread CTAs, two per SM
    ((8, 1, M_C2, False), (0, 0, 0, None)),     # three-launch: simhash -> probe -> attend_mma (stream-K)
    ((16, 1, M_C2, False), (0, 0, 0, None)),
    ((32, 1, M_C2, False), (0, 0, 0, None)),
    ((8, 1, M_LONG, True), (0, 0, 0, None)),    # beam and shared long-generation lines
    ((4, 4, M_C2, False), (1, 1, 1, 4)),        # verification: the fused T-token kernel, 128 resident clusters per wave
    ((8, 4, M_C2, False), (0, 0, 1, 8)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("shape,want", PATHS, ids=[f"B{s[0]}-T{s[1]}{'-spill' if s[3] else ''}" for s, _ in PATHS])
def test_measured_shapes_path(cuda_lib, shape, want):
    """Which sparse-layer path a step of each measured shape runs (Llama-3.1-8B heads, K10 L150, one slot)."""
    from magicpig_b200.ops import Context
    skip_unless_132_sms()
    B, T, M, spill = shape
    ctx = Context(KK, LL, 2, HQ, HKV, d, B, M, NS, NL, GEN, dense_layers=[0], device=DEV, max_query_tokens=T, num_contexts=1,
                  shared_spill=spill)
    got = [ctx.get_info("fused_applicable"), ctx.get_info("fused_cluster_waves")]
    g = torch.Generator(device=DEV).manual_seed(B)
    ctx.set_hash_func(synth.make_hash_func(d, KK, LL, seed=1).to(DEV))
    key = torch.randn((HKV, 300, d), generator=g, device=DEV).bfloat16()
    ctx.attn_fill(1, 0, key, key, key.float().norm(dim=-1))
    ctx.lsh_build(1, 0, ctx.hash_keys(key))
    for b in range(1, B):
        ctx.fork(0, b)
    for b in range(B):
        ctx.window_fill(1, b, torch.zeros((HKV, d), dtype=torch.bfloat16, device=DEV), key[:, :NS + NL].contiguous(),
                        key[:, :NS + NL].contiguous())
    q = torch.randn((B, T, HQ, d), generator=g, device=DEV).bfloat16()
    kv = torch.randn((B, T, HKV, d), generator=g, device=DEV).bfloat16()
    if T == 1:
        ctx.plan()
        ctx.decode(1, q[:, 0].contiguous(), kv[:, 0].contiguous(), kv[:, 0].contiguous())
    else:
        ctx.plan(T)
        ctx.decode_tokens(1, T, q, kv, kv)
    got.append(ctx.get_info("last_decode_fused"))
    got.append(ctx.get_info("tokens_cluster_waves") if T > 1 else None)
    assert tuple(got) == want, f"B={B} T={T}: (applicable, waves, fused, token waves) = {tuple(got)}"


# ---- 2./3. sparse cases ----------------------------------------------------------------------------------------------------
def sparse_case(label, regime, B, C=1, lens=LENS, place="key", T=1, parents=None, heads=None, fused=True, M=M_C2, gen=GEN,
                kreg=0, n=N_C2):
    """Generate, self-check, run one step and check it.  Fused steps run as the measured lines run them, with save_mask = 0
    (the CTAs list their selection in the carved extra row buffers); their codes and lists come from a save_mask = 1 twin
    filled identically, which must sample the same counts.  The three-launch path always writes its lists."""
    save_mask = 0 if fused else 1
    c = make_batch(regime, B, C=C, n=n, T=T, lens=lens, place=place, seed=seed_of(label, regime, place, kreg), parents=parents)
    moved = check_inputs(c, parents, heads)
    print(f"{label}: perturbations move the output by " + ", ".join(f"{k} {v:.2e}" for k, v in moved.items()))
    ctx = batch_ctx(c, C=0 if B == 1 else C, M=M, gen=gen, kreg=kreg, save_mask=save_mask, t_max=T)
    r = step(ctx, c, parents, lists=bool(save_mask))
    assert r["fused"] == int(fused), f"{label}: last_decode_fused = {r['fused']}"
    if not save_mask:
        tw = batch_ctx(c, C=0 if B == 1 else C, M=M, gen=gen, kreg=kreg, save_mask=1, t_max=T)
        rt = step(tw, c, parents)
        assert rt["fused"] == 1, f"{label}: the twin did not run the fused kernel"
        assert torch.equal(r["nnz"], rt["nnz"]), f"{label}: save_mask = 0 sampled other counts than its twin"
        r.update(res=rt["res"], codes=rt["codes"])
        del tw
    sets = check_codes_lists(c, r)
    return check_outputs(c, r, sets, label, parents, heads)


@pytest.mark.gpu
@pytest.mark.parametrize("kreg", [0, 1])
@pytest.mark.parametrize("regime", ["R1", "R2", "R4"])
def test_bench_config(cuda_lib, regime, kreg):
    """bench.py's configuration: B = 1 at C2 with save_mask = 0 (the CTAs list their selection in the carved extra row
    buffers), a full 324-row window."""
    sparse_case(f"bench {regime} kreg{kreg}", regime, 1, lens=(324,), kreg=kreg)


@pytest.mark.gpu
def test_shared_two(cuda_lib):
    sparse_case("shared B2", "R1", 2, lens=(69, 324))


@pytest.mark.gpu
@pytest.mark.parametrize("kreg", [0, 1])
@pytest.mark.parametrize("regime", ["R2", "R4"])
def test_shared_four(cuda_lib, regime, kreg):
    """Four requests on one slot: the fused kernel in 512-thread CTAs, ragged windows."""
    sparse_case(f"shared B4 {regime} kreg{kreg}", regime, 4, kreg=kreg)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["R1", "R2", "R4"])
def test_shared_eight(cuda_lib, regime):
    """Eight requests on one slot: the three-launch path, ragged windows."""
    sparse_case(f"shared B8 {regime}", regime, 8, fused=False)


@pytest.mark.gpu
def test_two_documents(cuda_lib):
    """Two slots holding different documents, requests bound 0, 1, 0, 1, ...: each attends over its own slot's store."""
    sparse_case("two documents B8", "R1", 8, C=2, fused=False)


@pytest.mark.gpu
def test_wide_batch(cuda_lib):
    """B = 32 on one slot: 1 024 heads in one step, the stream-K attend kernel at its widest.  Every head's codes and lists;
    fp64 outputs on four heads per request (rotating over the kv-groups), 128 heads.  R1: the sampled half carries nearly all of
    every head's mass, and dropping it must move every checked head by 10x the bar, so a lost or misweighted part shows."""
    heads = torch.zeros((32, HQ), dtype=torch.bool)
    for b in range(32):
        heads[b, [(b + 9 * j) % HQ for j in range(4)]] = True
    sparse_case("wide B32", "R1", 32, heads=heads, fused=False)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("regime,place", [("R2", "key"), ("R4", "win")], ids=["R2", "R4win"])
def test_long_windows(cuda_lib, regime, place, B):
    """generation_buffer 4 104: windows of 4 000 ... 4 172 rows (R2: the sinks thousands of rows before the query; R4: the
    dominant row in each window's last tile)."""
    lens = (4172,) if B == 1 else LONG_LENS
    sparse_case(f"long windows B{B} {regime}", regime, B, lens=lens, place=place, gen=LONG_GEN, fused=(B == 1))


@pytest.mark.gpu
@pytest.mark.parametrize("tree", [False, True], ids=["chain4", "tree8"])
def test_verification(cuda_lib, tree):
    """B = 8, a T = 4 chain or an 8-node tree after plan(T): every token against fp64 under the causal / ancestor mask, ragged
    windows; the fused T-token kernel in several waves."""
    T, parents = (8, [TREE] * 8) if tree else (4, None)
    sparse_case(f"verification B8 {'tree8' if tree else 'T4'}", "R2" if tree else "R4", 8, T=T, parents=parents)


# ---- after a shared spill ---------------------------------------------------------------------------------------------------
SPILLED = (40, 67, 101, 133, 170, 199, 230, 255)   # rows each request moves into the slot (window = NS + NL + these)


@pytest.mark.gpu
def test_after_shared_spill(cuda_lib):
    """B = 8 on one slot with shared_spill at the long-generation geometry (M = 131 072, generation_buffer 256).  Every request
    has grown its window by a different number of tokens (40 ... 255), decodes a step, spills; then a step with queries near
    its own spilled keys, a fork of a request that spilled, and one more step.  Each request against fp64 over the prompt, the
    private keys IT spilled and its remaining window.  The spilled rows are read back; their fp64 codes may differ from the
    codes the spill merged into the tables only where a projection is within rounding of zero, and the lists are restated
    over the merged codes."""
    B = 8
    c = make_batch("R1", B, lens=tuple(NS + NL + x for x in SPILLED), seed=seed_of("spill"))
    # window row NS + 3 (spilled by every request) is one row plus a little noise per request: a query near a request's own
    # copy is near every other request's copy too, so a request that saw another's private keys would attend to them
    gr = torch.Generator(device=DEV).manual_seed(4)
    for b in range(B):
        c["win_k"][b][:, NS + 3] = (c["win_k"][0][:, NS + 3].double()
                                    + 0.3 * torch.randn((HKV, d), generator=gr, device=DEV, dtype=torch.float64)).bfloat16()
    check_inputs(c)
    ctx = batch_ctx(c, M=M_LONG, shared_spill=True)
    r = step(ctx, c)
    assert r["fused"] == 0
    check_outputs(c, r, check_codes_lists(c, r), "before spill B8")
    for b in range(B):   # the step's token joins the window
        c["win_k"][b] = torch.cat([c["win_k"][b], (c["k_new"][b, 0] - avg_of(c, b))[:, None]], dim=1)
        c["win_v"][b] = torch.cat([c["win_v"][b], c["v_new"][b, 0][:, None]], dim=1)
    got = ctx.spill_window()
    assert got.tolist() == list(SPILLED)
    n, st = c["n"], c["slots"][0]
    total = n + sum(SPILLED)
    k_st, v_st, kn_st = ctx.read_cache(1)
    bits = lambda x: x.contiguous().view(torch.int16)   # noqa: E731
    assert torch.equal(bits(k_st[0, :, :n]), bits(st["key"])) and torch.equal(bits(v_st[0, :, :n]), bits(st["value"])), \
        "the spill changed the prompt's records"
    assert torch.equal(kn_st[0, :, :n], st["kn"]), "the spill changed the prompt's key norms"
    off = n
    for b in range(B):   # a slot's new keys go in request order; each request keeps its sinks and newest NL rows
        mk, mv = c["win_k"][b][:, NS:NS + SPILLED[b]], c["win_v"][b][:, NS:NS + SPILLED[b]]
        assert torch.equal(bits(k_st[0, :, off:off + SPILLED[b]]), bits(mk)), f"request {b}: spilled keys"
        assert torch.equal(bits(v_st[0, :, off:off + SPILLED[b]]), bits(mv)), f"request {b}: spilled values"
        kn = kn_st[0, :, off:off + SPILLED[b]]   # bf16(||k||) widened to fp32, as fill() stores
        norm = mk.double().norm(dim=-1)
        assert torch.equal(kn.bfloat16().float(), kn) and bool(((kn.double() - norm).abs() <= 2.0 ** -8 * norm).all()), \
            f"request {b}: spilled key norms"
        off += SPILLED[b]
        c["win_k"][b] = torch.cat([c["win_k"][b][:, :NS], c["win_k"][b][:, NS + SPILLED[b]:]], dim=1)
        c["win_v"][b] = torch.cat([c["win_v"][b][:, :NS], c["win_v"][b][:, NS + SPILLED[b]:]], dim=1)
    # the spilled keys' codes: fp64 from the rows read back; the tables hold the context's own hash of them, which may differ
    # only within rounding of a zero projection
    rows = k_st[0, :, n:total].contiguous()
    ours, theirs = key_codes(rows, c["hf"], KK, LL), ctx.hash_keys(rows)
    bad = torch.nonzero(ours != theirs)
    if bad.shape[0]:
        kk = rows[bad[:, 0], bad[:, 2]].double()
        cols = bad[:, 1, None] * KK + torch.arange(KK, device=DEV)[None]
        margin = (c["hf"].double().t()[cols] * kk[:, None]).sum(-1).abs().min(dim=-1).values
        assert float(margin.max()) < SIMHASH_EPS * float(rows.float().norm(dim=-1).mean()), float(margin.max())
    st.update(key=k_st[0, :, :total], value=v_st[0, :, :total], kn=kn_st[0, :, :total], kcodes=torch.cat([st["kcodes"], theirs], -1))
    spans, off = [], n
    for b in range(B):
        spans.append((off, off + SPILLED[b]))
        off += SPILLED[b]
    vis = [[s] for s in spans]
    g = torch.Generator(device=DEV).manual_seed(3)

    def masks(spans_of):
        out = []
        for b in range(B):
            m = torch.zeros(total, dtype=torch.bool, device=DEV)
            m[:n] = True
            for lo, hi in spans_of[b]:
                m[lo:hi] = True
            out.append(m)
        return out

    def private_step(label):
        c["vis"] = masks(vis)
        # queries near one of the request's own spilled keys, so that private keys are sampled
        near = torch.stack([st["key"][:, vis[b][0][0] + 3] for b in range(B)]).double()          # (B, Hkv, d)
        c["q"] = (near.repeat_interleave(c["G"], 1)[:, None] + 0.25 * torch.randn((B, 1, HQ, d), generator=g, device=DEV,
                                                                                   dtype=torch.float64)).bfloat16()
        c["k_new"] = (torch.randn((B, 1, HKV, d), generator=g, device=DEV, dtype=torch.float64)
                      + torch.stack([st["mu"]] * B).reshape(B, 1, HKV, d)).bfloat16()
        c["v_new"] = torch.randn((B, 1, HKV, d), generator=g, device=DEV).bfloat16()
        rr = step(ctx, c)
        assert rr["fused"] == 0, f"{label}: last_decode_fused = {rr['fused']}"
        sets = check_codes_lists(c, rr)
        # the private-key filter is visible: seeing every request's spilled keys, or none of its own, moves each request
        o, _ = restate_batch(c, rr["codes"], sets=sets)
        own = c["vis"]
        for name, other in (("sees_all_private", masks([spans] * B)), ("sees_no_private", masks([[]] * B))):
            c["vis"] = other
            alt, _ = restate_batch(c, rr["codes"])
            per_req = [rel_heads(alt[b], o[b]) for b in range(B)]
            assert min(per_req) >= 10 * BAR, f"{label}: '{name}' moves a request by {min(per_req):.2e} only"
            print(f"{label}: {name} moves every request by >= {min(per_req):.2e}")
        c["vis"] = own
        check_outputs(c, rr, sets, label)
        for b in range(B):
            private = rr["res"][b, 0, :, :][torch.arange(rr["res"].shape[-1], device=DEV)[None] < rr["nnz"][b, 0][:, None]]
            assert bool((private >= n).any()), f"request {b} sampled none of its spilled keys"
            c["win_k"][b] = torch.cat([c["win_k"][b], (c["k_new"][b, 0] - avg_of(c, b))[:, None]], dim=1)
            c["win_v"][b] = torch.cat([c["win_v"][b], c["v_new"][b, 0][:, None]], dim=1)

    private_step("after spill B8")
    ctx.fork(2, 5)   # request 5 continues request 2: its window and the private keys 2 sees
    vis[5] = list(vis[2])
    c["win_k"][5], c["win_v"][5] = c["win_k"][2].clone(), c["win_v"][2].clone()
    private_step("after spill and fork B8")


# ---- dense layers in shared-prefix mode --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 4])
@pytest.mark.parametrize("B", [8, 32])
@pytest.mark.parametrize("regime", ["R2", "R4"])
def test_dense_shared_prefix(cuda_lib, regime, B, T):
    """dense_tail_rows 16 over one 98 000-row prompt in the slot: each request kept a different number of rows of two earlier
    4-token steps (ragged tails); the step against fp64 over the prompt plus that request's own tail.  The dense kernel puts up
    to max(1, 32 / (T * G)) requests of one slot in a chunk (dense_slot_chunks), so these shapes form 1 (B = 8, T = 1), 4 or 16
    chunks; the library reports no chunk count, so this reading of the kernel is not asserted."""
    from magicpig_b200.ops import Context
    P = 98000
    c = make_dense_slots(regime, B, P, T, seed=seed_of("dense", regime, B, T))
    o, moved = check_dense_inputs(c)
    ctx = Context(4, 8, 2, HQ, HKV, d, B, M_C2, NS, NL, GEN, dense_layers=[0], alloc_dense_kv=True, device=DEV,
                  max_query_tokens=4, num_contexts=1, dense_tail_rows=16)
    ctx.set_option("out_f32", 1)
    ctx.set_hash_func(synth.make_hash_func(d, 4, 8, seed=1).to(DEV))
    small = torch.randn((HKV, 64, d), generator=torch.Generator(device=DEV).manual_seed(1), device=DEV).bfloat16()
    ctx.attn_fill(1, 0, small, small, small.float().norm(dim=-1))
    ctx.lsh_build(1, 0, ctx.hash_keys(small))
    ctx.window_fill(1, 0, torch.zeros((HKV, d), dtype=torch.bfloat16, device=DEV), small, small)
    ctx.dense_fill(0, 0, c["dk"].contiguous(), c["dv"].contiguous(), P)
    for b in range(1, B):
        ctx.fork(0, b)
    for pq, pk, pv, drop in c["pre"]:
        ctx.plan(4)
        ctx.dense_decode_tokens(0, 4, pq, pk, pv)
        ctx.rewind(torch.tensor(drop, dtype=torch.int32, device=DEV))
    if T == 1:
        ctx.plan()
        out = ctx.dense_decode(0, c["q"][:, 0].contiguous(), c["k"][:, 0].contiguous(), c["v"][:, 0].contiguous())
    else:
        ctx.plan(T)
        out = ctx.dense_decode_tokens(0, T, c["q"], c["k"], c["v"])
    o32 = ctx.last_out_f32()
    assert ctx.error_flags() == 0
    worst = rel_heads(o32, o)
    label = f"dense B{B} T{T} {regime}"
    print(f"{label}: perturbations " + ", ".join(f"{k} {v:.2e}" for k, v in moved.items())
          + f"; largest relative head error {worst:.2e} ({worst / BAR:.1%} of the bar)")
    assert worst <= BAR, f"{label}: fp32 output differs from fp64 by {worst:.3e} relative"
    assert torch.equal(out.cpu().view(torch.int16).int().reshape(-1) & 0xFFFF, bf16_half_up(o32).reshape(-1))
