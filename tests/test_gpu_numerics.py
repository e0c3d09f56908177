"""Attention kernels against an fp64 restatement on model-shaped inputs (`-m gpu`).

The other GPU files mostly check a path against a twin (T tokens against T single steps, a fork against a private copy) and
give the absolute check i.i.d. Gaussian inputs, on which the key mean is near zero, the window carries a few per cent of the
mass and the softmax is flat.  A kernel that forgot to centre the new key, dropped a window row or skipped a rescale passes
there.  The inputs here are shaped like a model's instead, one knob per regime:

  R1  key mean: keys = mu + noise with |mu| four times the per-key noise; the store and the window hold centred rows, the new
      tokens carry mu and the kernel must subtract avg_k itself;
  R2  sinks: the num_sink_tokens first window rows (and the new token) are aligned with every query of the group, so the window
      holds >= 90 % of the mass;
  R3  balanced: each query is scaled so that the window's share of the merged mass is 0.35 or 0.65;
  R4  large logits: queries x 16 (scores span >= 40 nats) and one dominant key, placed first or last in the store;
  R5  parallel keys: a few stored keys are exact bf16 multiples of a query, so cs rounds past 1 and the clamp is taken.

The restatement (`restate`) takes the sample set from collision counts over the GPU's own query codes (checked first against
an fp64 projection with the margin rule of test_simhash), clamps cos to [-1, 1], applies the LSH weight, attends the window
rows plus bf16(k_new - avg_k) under the causal / ancestor mask of the step, and merges the two halves by their base-2 LSEs,
all in fp64.  One exception: the weight 1 - (1-p)^(L-1) (Lp + 1 - p) is evaluated in the reference's fp32 order (as the C
oracle does), because for w <~ 1e-4 its fp32 cancellation is part of the reference's definition of the output, and a kernel
computing it in fp32 cannot be held to the fp64 value there.

Every generator checks, before any GPU call, that its inputs can tell a broken kernel from a correct one: a named perturbation
of the restatement (`SELF_CHECK`) must move the output by at least 10x the 1e-3 bar.
"""
import math
import zlib

import pytest
import torch

import oracle
from magicpig_b200 import synth
from tests.test_gpu_parity import SIMHASH_EPS, assert_1e3_f32
from tests.test_gpu_tokens import bf16_half_up

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
d, NS, NL, GEN = 128, 4, 64, 32
BAR = 1e-3
TILE = 16                      # rows per tile of the restatement's online softmax (the sparse kernels' tile)
SELF_CHECK = {"R1": "uncentred", "R2": "drop_newest", "R3": "ln_merge", "R4": "skip_rescale"}


# ------------------------------------------------------------------------------------------------
# fp64 restatement
# ------------------------------------------------------------------------------------------------
def lsh_weight(cs: torch.Tensor, K: int, L: int) -> torch.Tensor:
    """Collision weight of keys at cosine cs (fp64, clamped): theta and p in fp64, then the reference's fp32 expression order
    for 1 - (1-p)^(L-1) (L p + 1 - p) (its cancellation below w ~ 1e-4 is part of the reference's output)."""
    theta = torch.arccos(cs.clamp(-1.0, 1.0))
    proba = (1.0 - theta / math.pi).float()
    p = proba ** K
    qq = 1.0 - p
    w = 1.0 - qq ** (L - 1) * (L * p + qq)
    return w.double()


def sample_scores(q: torch.Tensor, k: torch.Tensor, kn: torch.Tensor, K: int, L: int) -> torch.Tensor:
    """z of sampled rows: s / sqrt(d) - log(w + 1e-4).  q (d,) bf16, k (m, d) bf16, kn (m,) fp32 stored norms."""
    s = k.double() @ q.double()
    cs = s / (q.double().norm() * kn.double())
    return s / math.sqrt(d) - torch.log(lsh_weight(cs, K, L) + 1e-4)


def softmax_state(z: torch.Tensor, v: torch.Tensor, skip_rescale: bool = False, tile: int = TILE):
    """(o, base-2 LSE) of rows with scores z over values v (fp64).  skip_rescale: what a tiled online softmax computes when it
    leaves out the rescale of the running state at one tile (a kernel bug the inputs must expose): every row before that tile
    keeps a weight too large by e^jump, jump = how far the running max rises there.  The tile is the one where that matters
    most (largest excess weight)."""
    if z.numel() == 0 or not bool(torch.isfinite(z).any()):
        return torch.zeros(v.shape[-1], dtype=torch.float64, device=z.device), -math.inf
    v = v.double()
    m = z.max()
    e = torch.exp(z - m)
    if skip_rescale:
        pad = torch.full((-len(z) % tile,), -math.inf, dtype=z.dtype, device=z.device)
        run = torch.cummax(torch.cat([z, pad]).reshape(-1, tile).max(dim=1).values, 0).values
        if len(run) > 1:
            jumps = (run[1:] - run[:-1]).clamp(max=700.0)
            before = torch.cumsum(torch.cat([e, pad.exp()]).reshape(-1, tile).sum(dim=1), 0)[:-1]   # mass before tiles 1..
            t = int((torch.expm1(jumps) * before).argmax()) + 1
            e[: t * tile] *= math.exp(float(jumps[t - 1]))
    return (e @ v) / e.sum(), float((torch.log(e.sum()) + m) / math.log(2))


def merge2(o_a, lse_a, o_b, lse_b, natural: bool = False):
    """Merge two softmax states by base-2 LSE (natural=True: the bug of treating them as natural-log values)."""
    m = max(lse_a, lse_b)
    if m == -math.inf:
        return torch.zeros_like(o_a)
    f = math.exp if natural else (lambda x: 2.0 ** x)
    a, b = f(lse_a - m), f(lse_b - m)
    return (a * o_a + b * o_b) / (a + b)


def sample_sets(c, qcodes: torch.Tensor):
    """Index lists (ascending) of the keys that collide in >= 2 tables: qcodes int32 (B, T, Hq, L) -> [b][t][h] LongTensor."""
    B, T, Hq = qcodes.shape[:3]
    out = []
    for b in range(B):
        rows = []
        for t in range(T):
            cnt = oracle.collision_counts(c["kcodes"][b].contiguous(), qcodes[b, t].contiguous(), c["G"])
            rows.append([torch.nonzero(cnt[h] > 1).flatten() for h in range(Hq)])
        out.append(rows)
    return out


def cpu_codes(c) -> torch.Tensor:
    B, T, Hq = c["q"].shape[:3]
    codes, _ = oracle.simhash(c["q"].reshape(-1, d).contiguous(), c["hf"], c["K"], c["L"])
    return codes.reshape(B, T, Hq, c["L"])


def visible(parents, b, t):
    """Earlier step tokens token t attends to besides itself: all before it (chain) or its ancestors (tree)."""
    if parents is None:
        return list(range(t))
    anc, j = [], parents[b][t]
    while j >= 0:
        anc.append(j)
        j = parents[b][j]
    return anc[::-1]


def restate(c, qcodes=None, parents=None, variant=None, sets=None):
    """fp64 output of the sparse decode step of case c: (o (B, T, Hq, d), lse_s (B, T, Hq) base-2 LSE of the sampled half,
    share (B, T, Hq) the window's share of the merged mass).  variant: one of SELF_CHECK's perturbations, or None."""
    q, G, K, L = c["q"], c["G"], c["K"], c["L"]
    B, T, Hq = q.shape[:3]
    if sets is None:
        sets = sample_sets(c, cpu_codes(c) if qcodes is None else qcodes)
    o = torch.zeros((B, T, Hq, d), dtype=torch.float64)
    lse_s = torch.full((B, T, Hq), -math.inf, dtype=torch.float64)
    share = torch.zeros((B, T, Hq), dtype=torch.float64)
    for b in range(B):
        for t in range(T):
            vis = visible(parents, b, t)
            for g in range(c["Hkv"]):
                new = c["k_new"][b, :, g] if variant == "uncentred" else c["k_new"][b, :, g] - c["avg"][b, g]
                wk = torch.cat([c["win_k"][b, g], new[vis], new[t:t + 1]])
                wv = torch.cat([c["win_v"][b, g], c["v_new"][b, vis, g], c["v_new"][b, t:t + 1, g]])
                if variant == "drop_newest":
                    wk, wv = wk[:-1], wv[:-1]
                for h in range(g * G, (g + 1) * G):
                    qh = q[b, t, h]
                    idx = sets[b][t][h]
                    zs = sample_scores(qh, c["key"][b, g, idx], c["kn"][b, g, idx], K, L)
                    zw = (wk.double() @ qh.double()) / math.sqrt(d)
                    if variant == "skip_rescale":
                        o[b, t, h], _ = softmax_state(torch.cat([zw, zs]), torch.cat([wv, c["value"][b, g, idx]]), True)
                        continue
                    o_s, l_s = softmax_state(zs, c["value"][b, g, idx])
                    o_w, l_w = softmax_state(zw, wv)
                    o[b, t, h] = merge2(o_w, l_w, o_s, l_s, natural=(variant == "ln_merge"))
                    lse_s[b, t, h] = l_s
                    share[b, t, h] = 1.0 / (1.0 + 2.0 ** (l_s - l_w)) if l_s > -math.inf else 1.0
    return o, lse_s, share


def rel_head(a: torch.Tensor, o: torch.Tensor) -> float:
    """max over heads of max|a - o| / max|o| (the bar's metric)."""
    a, o = a.double().reshape(-1, d), o.double().reshape(-1, d)
    return float(((a - o).abs().amax(-1) / o.abs().amax(-1).clamp_min(1e-30)).max())


def self_check(c, name, o, run):
    """The regime's named perturbation of the restatement must move the output by >= 10x the bar."""
    moved = rel_head(run(SELF_CHECK[name]), o)
    assert moved >= 10 * BAR, f"{name}: inputs are insensitive, '{SELF_CHECK[name]}' moves the output by {moved:.2e} only"
    return moved


# ------------------------------------------------------------------------------------------------
# generator
# ------------------------------------------------------------------------------------------------
def _unit(g, *shape):
    u = torch.randn((*shape, d), generator=g, dtype=torch.float64)
    return u / u.norm(dim=-1, keepdim=True)


def make_case(regime, B, Hq, Hkv, n, K, L, seed, T=1, place="last", parents=None):
    """Sparse-layer inputs of one regime (R1..R5, R4 with the dominant key `place`d first or last in the store), tuned on the
    CPU codes.  Returns a dict of CPU tensors: q (B,T,Hq,d), key/value (B,Hkv,n,d) centred store, kn, avg (B,Hkv,d), kcodes,
    win_k/win_v (B,Hkv,NS+NL,d) centred window, k_new/v_new (B,T,Hkv,d) as the model produces them (uncentred)."""
    g = torch.Generator().manual_seed(seed)
    G, W = Hq // Hkv, NS + NL
    hf = synth.make_hash_func(d, K, L, seed=seed + 1)
    u = _unit(g, B, Hkv)                                                    # one direction per kv group
    rd = math.sqrt(d)
    qn = 0.5 if regime == "R4" else 1.0
    q = qn * torch.randn((B, T, Hq, d), generator=g, dtype=torch.float64) + rd * u.repeat_interleave(G, 1)[:, None]
    mu = torch.zeros((B, Hkv, 1, d), dtype=torch.float64)
    if regime == "R1":   # |mu| ~ 4 |noise|, partly along the queries (which is what makes an uncentred key visible)
        mu = 4.0 * (0.8 * torch.randn((B, Hkv, 1, d), generator=g, dtype=torch.float64) + 0.6 * rd * u[:, :, None])
    key = torch.randn((B, Hkv, n, d), generator=g, dtype=torch.float64)
    if regime != "R4":   # a share of the keys clusters around the group direction, so that K10 L150 samples some of them
        pull = (torch.rand((B, Hkv, n, 1), generator=g) < 0.125) * torch.rand((B, Hkv, n, 1), generator=g, dtype=torch.float64) * 1.2
        key = key + pull * rd * u[:, :, None]
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
    c = dict(B=B, Hq=Hq, Hkv=Hkv, G=G, n=n, K=K, L=L, hf=hf, q=q.bfloat16(), key=key, value=value, avg=avg.reshape(B, Hkv, d),
             win_k=win_k, win_v=win_v, k_new=k_new.bfloat16(), v_new=v_new, regime=regime)
    if regime == "R5":   # stored keys that are exact power-of-two multiples of a query whose bf16 norm rounds down
        q0 = c["q"][:, 0]
        for b in range(B):
            for h in range(Hq):
                qn32 = q0[b, h].float().norm()
                for j, sc in enumerate((1.0, 2.0, 0.5)):
                    kk = (q0[b, h].float() * sc).bfloat16()
                    if float(kk.norm().float()) < float(qn32) * sc:   # the stored bf16 norm rounds down: cs > 1 in fp32
                        key[b, h // G, (h * 7 + 101 * j) % n] = kk
    c["key"] = key
    c["kn"] = key.norm(p=2, dim=-1).float()                                   # norm of the bf16 keys, bf16-rounded (reference)
    c["kcodes"] = synth.hash_keys(key, hf, K, L)
    _tune(c, regime, u, place, parents)
    return c


def _parts(c, sets, b, t, h, win_extra=None):
    """Per-row raw dot products and LSH offsets of one head (for the knob tuning): sampled s, -log(w) and window s."""
    g = h // c["G"]
    qh = c["q"][b, t, h].double()
    idx = sets[b][t][h]
    s = c["key"][b, g, idx].double() @ qh
    cs = s / (qh.norm() * c["kn"][b, g, idx].double())
    off = -torch.log(lsh_weight(cs, c["K"], c["L"]) + 1e-4)
    wk = c["win_k"][b, g] if win_extra is None else torch.cat([c["win_k"][b, g], win_extra])
    return s / math.sqrt(d), off, (wk.double() @ qh) / math.sqrt(d)


def _tune(c, regime, u, place, parents):
    B, T, Hq, G = c["B"], c["q"].shape[1], c["Hq"], c["G"]
    rd = math.sqrt(d)
    if regime in ("R2", "R3"):
        # sink rows (and the new tokens) along the group direction; R2: strong enough that the window holds >= 90 % of the mass
        sets = sample_sets(c, cpu_codes(c))
        sigma = 2.0
        if regime == "R2":
            need = 0.0
            for b in range(B):
                for t in range(T):
                    for h in range(Hq):
                        s, off, sw = _parts(c, sets, b, t, h)
                        rest = torch.logsumexp(torch.cat([s + off, sw[NS:]]), 0)
                        a = float(c["q"][b, t, h].double() @ u[b, h // G])          # sink score per unit of sigma
                        need = max(need, (float(rest) + math.log(9 * 4) + 1.0 - math.log(NS)) / a)
            sigma = need
        sink = (sigma * rd * u).bfloat16()                                          # (B, Hkv, d)
        c["win_k"][:, :, :NS] = sink[:, :, None]
        c["k_new"] = (c["k_new"].double() * 0.25 + (sink.double() + c["avg"].double())[:, None]).bfloat16()
    if regime == "R3":
        # per query a scale lambda (bisection) for a window share of 0.35 / 0.65 alternately
        sets = sample_sets(c, cpu_codes(c))
        q = c["q"].double().clone()
        for b in range(B):
            for t in range(T):
                for h in range(Hq):
                    target = 0.35 if h % 2 == 0 else 0.65
                    new = (c["k_new"][b, visible(parents, b, t) + [t], h // G] - c["avg"][b, h // G])
                    s, off, sw = _parts(c, sets, b, t, h, win_extra=new)
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
        sets = sample_sets(c, cpu_codes(c))
        pos = 0 if place == "first" else c["n"] - 1
        unit_key = (rd * u).bfloat16()
        for b in range(B):
            for g in range(c["Hkv"]):
                c["key"][b, g, pos] = unit_key[b, g]
        c["kn"] = c["key"].norm(p=2, dim=-1).float()
        c["kcodes"] = synth.hash_keys(c["key"], c["hf"], c["K"], c["L"])
        sets = sample_sets(c, cpu_codes(c))
        deltas = []
        for b in range(B):
            for t in range(T):
                for h in range(Hq):
                    g = h // G
                    idx = sets[b][t][h]
                    if not bool((idx == pos).any()):
                        continue
                    s, off, sw = _parts(c, sets, b, t, h)
                    mine = idx == pos
                    rest = torch.logsumexp(torch.cat([(s + off)[~mine], sw]), 0)
                    deltas.append((float(rest - off[mine][0]) / float(s[mine][0])))
        assert len(deltas) * 2 >= B * T * Hq, "the dominant key is not sampled for most queries"
        delta = max(sorted(deltas)[len(deltas) // 2], 2.0 ** -6)
        for b in range(B):
            for g in range(c["Hkv"]):
                c["key"][b, g, pos] = (unit_key[b, g].double() * delta).bfloat16()
        c["kn"] = c["key"].norm(p=2, dim=-1).float()
        c["kcodes"] = synth.hash_keys(c["key"], c["hf"], c["K"], c["L"])
        c["dominant"] = pos


def check_case(c, parents=None):
    """The generator's self-checks (fp64, CPU codes, no GPU): the regime's property holds and its perturbation is visible."""
    regime = c["regime"]
    sets = sample_sets(c, cpu_codes(c))
    o, lse_s, share = restate(c, parents=parents, sets=sets)
    assert torch.isfinite(o).all()
    run = lambda v: restate(c, parents=parents, variant=v, sets=sets)[0]
    if regime == "R2":
        assert float(share.min()) >= 0.9, f"R2: window share {float(share.min()):.3f} < 0.9"
    if regime == "R3":
        assert 0.3 <= float(share.min()) and float(share.max()) <= 0.7, f"R3: window share in [{share.min():.3f}, {share.max():.3f}]"
    if regime == "R4":
        span = []
        for b in range(c["B"]):
            for t in range(c["q"].shape[1]):
                for h in range(c["Hq"]):
                    s, off, sw = _parts(c, sets, b, t, h)
                    z = torch.cat([s + off, sw])
                    span.append(float(z.max() - z.min()))
        assert min(span) >= 40.0, f"R4: scores span {min(span):.1f} nats only"
    if regime == "R5":
        hit = 0
        for b in range(c["B"]):
            for h in range(c["Hq"]):
                idx = sets[b][0][h]
                qh = c["q"][b, 0, h]
                cs = (c["key"][b, h // c["G"], idx].float() @ qh.float()) / (qh.float().norm() * c["kn"][b, h // c["G"], idx])
                hit += int((cs > 1.0).sum())
        assert hit > 0, "R5: no sampled key has an fp32 cosine past 1"
    if regime in SELF_CHECK:
        self_check(c, regime, o, run)
    return o


# ---- dense layers --------------------------------------------------------------------------------
def make_dense(regime, B, Hq, Hkv, P, T, seed, place="last", one_prompt=False):
    """Dense-layer inputs: prompt rows dk/dv (B, P, Hkv, d), q (B, T, Hq, d), step rows k/v (B, T, Hkv, d).
    R2: the first NS prompt rows and the step's keys lie along the group direction and hold >= 90 % of the mass;
    R4: queries x 16 and one dominant row at the first / last prompt row (place="new": the step's last key).
    one_prompt: every request has the same prompt (and query direction), as the requests bound to one context slot."""
    g = torch.Generator().manual_seed(seed)
    G = Hq // Hkv
    rd = math.sqrt(d)
    u = _unit(g, 1 if one_prompt else B, Hkv).expand(B, Hkv, d)
    q = 0.5 * torch.randn((B, T, Hq, d), generator=g, dtype=torch.float64) + rd * u.repeat_interleave(G, 1)[:, None]
    dk = torch.randn((1 if one_prompt else B, P, Hkv, d), generator=g, dtype=torch.float64).expand(B, P, Hkv, d).clone()
    dv = torch.randn((1 if one_prompt else B, P, Hkv, d), generator=g).bfloat16().expand(B, P, Hkv, d).clone()
    k = torch.randn((B, T, Hkv, d), generator=g, dtype=torch.float64)
    v = torch.randn((B, T, Hkv, d), generator=g).bfloat16()
    c = dict(B=B, Hq=Hq, Hkv=Hkv, G=G, P=P, regime=regime, place=place)
    if regime == "R2":
        qq = q.bfloat16().double()
        a = torch.einsum("bthd,bhd->bth", qq, u.repeat_interleave(G, 1)).min()
        rest = math.log(P + T) + 8.0                       # every other score is below 8 nats for these queries
        sigma = (rest + math.log(9 * 2)) / float(a)
        ns = min(NS, P)
        dk[:, :ns] = sigma * rd * u[:, None]
        k = 0.25 * k + sigma * rd * u[:, None]
    else:
        q = q * 16.0
        qq = q.bfloat16().double()
        pos = {"first": 0, "last": P - 1, "new": None}[place]
        rows = torch.cat([dk, k], dim=1)
        s = torch.einsum("btkgd,bnkd->btkgn", qq.reshape(B, T, Hkv, G, d), rows) / rd
        a = torch.einsum("btkgd,bkd->btkg", qq.reshape(B, T, Hkv, G, d), u)      # score of the row rd * u per unit of delta
        delta = float(((torch.logsumexp(s, -1) + 2.0) / a).median())               # ~90 % of the mass for the median query
        dom = delta * rd * u
        if pos is None:
            k[:, -1] = dom
        else:
            dk[:, pos] = dom
    c.update(q=q.bfloat16(), dk=dk.bfloat16(), dv=dv, k=k.bfloat16(), v=v)
    return c


def restate_dense(c, parents=None, variant=None):
    """fp64 output (B, T, Hq, d) of a dense step: prompt rows + the visible step rows (causal or ancestors) + the token."""
    B, T, Hq, G = c["B"], c["q"].shape[1], c["Hq"], c["G"]
    o = torch.zeros((B, T, Hq, d), dtype=torch.float64)
    for b in range(B):
        for t in range(T):
            rows = visible(parents, b, t) + [t]
            kk = torch.cat([c["dk"][b], c["k"][b, rows]])
            vv = torch.cat([c["dv"][b], c["v"][b, rows]])
            if variant == "drop_newest":
                kk, vv = kk[:-1], vv[:-1]
            if variant == "skip_rescale" and c.get("place") == "first":   # (order-free sum: visit the dominant row last)
                kk, vv = kk.flip(0), vv.flip(0)
            for h in range(Hq):
                z = (kk[:, h // G].double() @ c["q"][b, t, h].double()) / math.sqrt(d)
                if variant == "skip_rescale":   # row-granular, so that small P still has a rescale to skip
                    o[b, t, h], _ = softmax_state(z, vv[:, h // G], True, tile=1)
                else:
                    o[b, t, h], _ = softmax_state(z, vv[:, h // G])
    return o


def check_dense(c, parents=None):
    o = restate_dense(c, parents)
    variant = "drop_newest" if c["regime"] == "R2" else "skip_rescale"
    moved = rel_head(restate_dense(c, parents, variant), o)
    assert moved >= 10 * BAR, f"dense {c['regime']}: '{variant}' moves the output by {moved:.2e} only"
    return o


# ------------------------------------------------------------------------------------------------
# GPU side
# ------------------------------------------------------------------------------------------------
def check_codes(c, codes: torch.Tensor):
    """GPU query codes (B, T, Hq, L) against the fp64 projection of the query normalised as the reference does (bf16 norm, bf16
    quotient; oracle.simhash): a code may differ only where one of its K projections is within SIMHASH_EPS of zero
    (test_simhash's rule, no count allowance)."""
    ref, margin = oracle.simhash(c["q"].reshape(-1, d).contiguous(), c["hf"], c["K"], c["L"])
    bad = codes.reshape(ref.shape) != ref
    if bool(bad.any()):
        assert float(margin[bad].max()) < SIMHASH_EPS, f"{int(bad.sum())} query codes differ beyond rounding"


def check_lists(c, sets, nnz, res):
    B, T, Hq = nnz.shape
    for b in range(B):
        for t in range(T):
            for h in range(Hq):
                n_ = int(nnz[b, t, h])
                assert n_ == len(sets[b][t][h]), (b, t, h)
                assert torch.equal(res[b, t, h, :n_].long(), sets[b][t][h]), (b, t, h)


def sparse_ctx(c, impl=1, kreg=0, t_max=1, M=None, **opts):
    from magicpig_b200.ops import Context
    ctx = Context(c["K"], c["L"], 2, c["Hq"], c["Hkv"], d, c["B"], M or c["n"] + 256, NS, NL, GEN, dense_layers=[0],
                  device=DEV, max_query_tokens=t_max)
    for key, val in dict(decode_impl=impl, fused_kreg=kreg, save_mask=1, out_f32=1, **opts).items():
        ctx.set_option(key, val)
    ctx.set_hash_func(c["hf"].to(DEV))
    for b in range(c["B"]):
        ctx.attn_fill(1, b, c["key"][b].to(DEV).contiguous(), c["value"][b].to(DEV).contiguous(), c["kn"][b].to(DEV).contiguous())
        ctx.lsh_build(1, b, c["kcodes"][b].to(DEV).contiguous())
        ctx.window_fill(1, b, c["avg"][b].to(DEV).contiguous(), c["win_k"][b].to(DEV).contiguous(), c["win_v"][b].to(DEV).contiguous())
    return ctx


def run_step(ctx, c, parents=None):
    """One step of c's T tokens (T = 1: plan + decode); returns readouts shaped (B, T, Hq, ...)."""
    B, T, Hq = c["q"].shape[:3]
    if T == 1:
        ctx.plan()
        out = ctx.decode(1, c["q"][:, 0].contiguous().to(DEV), c["k_new"][:, 0].contiguous().to(DEV),
                         c["v_new"][:, 0].contiguous().to(DEV))
    else:
        ctx.plan(T, parents=None if parents is None else torch.tensor(parents, dtype=torch.int32, device=DEV))
        out = ctx.decode_tokens(1, T, c["q"].to(DEV), c["k_new"].to(DEV), c["v_new"].to(DEV))
    nnz, res = ctx.last_probe(want_results=True)
    return dict(out=out.cpu().reshape(B, T, Hq, d), o32=ctx.last_out_f32().cpu().reshape(B, T, Hq, d),
                codes=ctx.last_codes().cpu().reshape(B, T, Hq, -1), nnz=nnz.cpu().reshape(B, T, Hq),
                res=res.cpu().reshape(B, T, Hq, -1))


def check_step(c, r, parents=None):
    """Codes, index lists and nnz against fp64; fp32 output within 1e-3 of the restatement; bf16 output = fp32 rounded once."""
    check_codes(c, r["codes"])
    sets = sample_sets(c, r["codes"])
    check_lists(c, sets, r["nnz"], r["res"])
    o, lse_s, _ = restate(c, parents=parents, sets=sets)
    assert_1e3_f32(r["o32"].reshape(-1, d), o.reshape(-1, d))
    assert torch.equal(r["out"].view(torch.int16).int() & 0xFFFF, bf16_half_up(r["o32"]).reshape(r["out"].shape))
    return o, lse_s


SHAPES = [
    (1, 16, 4, 4096, 10, 150),     # clusters of 4
    (1, 4, 1, 1500, 8, 60),        # clusters of 8
    (1, 8, 1, 70000, 8, 40),       # two key segments
    (4, 32, 8, 2000, 8, 60),       # 128 heads, one CTA each
]
REGIMES = [("R1", "last"), ("R2", "last"), ("R3", "last"), ("R4", "first"), ("R4", "last"), ("R5", "last")]
_cases = {}


def case(regime, place, shape, T=1):
    key = (regime, place, shape, T)
    if key not in _cases:
        B, Hq, Hkv, n, K, L = shape
        c = make_case(regime, B, Hq, Hkv, n, K, L, seed=zlib.crc32(repr(key).encode()) % 10000, T=T, place=place)
        check_case(c)
        _cases[key] = c
    return _cases[key]


# ---- fused single-token decode, three-launch path, stand-alone gather kernel --------------------------------------------
@pytest.mark.parametrize("kreg", [0, 1])
@pytest.mark.parametrize("shape", SHAPES, ids=["c4", "c8", "seg2", "cta1"])
@pytest.mark.parametrize("regime,place", REGIMES, ids=[f"{r}{p[0]}" if r == "R4" else r for r, p in REGIMES])
def test_fused_decode_regimes(cuda_lib, regime, place, shape, kreg):
    c = case(regime, place, shape)
    ctx = sparse_ctx(c, impl=1, kreg=kreg)
    r = run_step(ctx, c)
    assert ctx.get_info("last_decode_fused") == 1
    check_step(c, r)


@pytest.mark.parametrize("tma", [0, 1])
@pytest.mark.parametrize("regime,place", REGIMES, ids=[f"{r}{p[0]}" if r == "R4" else r for r, p in REGIMES])
def test_three_launch_and_gather_regimes(cuda_lib, regime, place, tma):
    """decode_impl 0 (SimHash | probe | attend) and the stand-alone gather kernel (mpig_attention_wrapper), whose base-2 LSE
    (mve row 1) must match the sampled half's fp64 LSE."""
    c = case(regime, place, SHAPES[0])
    ctx = sparse_ctx(c, impl=0, attend_tma=tma)
    r = run_step(ctx, c)
    assert ctx.get_info("last_decode_fused") == 0
    _, lse_s = check_step(c, r)
    H = c["B"] * c["Hq"]
    res = torch.zeros((H, ctx.M), dtype=torch.int32)
    for i in range(H):
        res[i, : int(r["nnz"].reshape(-1)[i])] = r["res"].reshape(H, -1)[i, : int(r["nnz"].reshape(-1)[i])]
    out = torch.zeros((H, d), dtype=torch.bfloat16, device=DEV)
    mve = torch.zeros((2, H), dtype=torch.float32, device=DEV)
    q = c["q"][:, 0].reshape(H, d).contiguous()
    ctx.attention_wrapper(1, c["K"], c["L"], out, mve, q.to(DEV), q.float().norm(dim=-1).to(DEV), res.to(DEV),
                          r["nnz"].reshape(-1).contiguous().to(DEV))
    o32 = ctx.last_out_f32().cpu()
    sets = sample_sets(c, r["codes"])
    for i in range(H):
        b, h = divmod(i, c["Hq"])
        idx = sets[b][0][h]
        o_s, l_s = softmax_state(sample_scores(q[i], c["key"][b, h // c["G"], idx], c["kn"][b, h // c["G"], idx], c["K"], c["L"]),
                                 c["value"][b, h // c["G"], idx])
        assert_1e3_f32(o32[i][None], o_s[None])
        if l_s == -math.inf:
            assert float(mve[1, i]) == -math.inf
        else:
            assert abs(float(mve[1, i]) - l_s) <= BAR * max(1.0, abs(l_s)), (i, float(mve[1, i]), l_s)


# ---- T-token steps and a tree ---------------------------------------------------------------------------------------------
TREE = [-1, 0, 0, 1, 1, 2, 3, 3]


@pytest.mark.parametrize("kreg", [0, 1])
@pytest.mark.parametrize("T,tree", [(3, False), (8, False), (8, True)], ids=["T3", "T8", "tree8"])
@pytest.mark.parametrize("regime", ["R1", "R2", "R3", "R4"])
def test_tokens_regimes(cuda_lib, regime, T, tree, kreg):
    """Every token of a step of T tokens (or node of an 8-node branching tree) directly against fp64, with the causal or
    ancestor mask over the step's rows."""
    B, Hq, Hkv, n, K, L = 2, 8, 2, 3000, 8, 60
    parents = [TREE] * B if tree else None
    c = make_case(regime, B, Hq, Hkv, n, K, L, seed=31 + T + 7 * tree, T=T, parents=parents)
    check_case(c, parents)
    ctx = sparse_ctx(c, kreg=kreg, t_max=T)
    check_step(c, run_step(ctx, c, parents), parents)


def test_decode_after_spill_r1(cuda_lib):
    """Under a large key mean, spilled window rows keep their centring: decode after spill_window against fp64 over the store
    as it now is (its keys, norms and the GPU's codes of them)."""
    B, Hq, Hkv, n, K, L = 2, 8, 2, 1500, 7, 40
    c = make_case("R1", B, Hq, Hkv, n, K, L, seed=5)
    check_case(c)
    ctx = sparse_ctx(c)
    g = torch.Generator().manual_seed(6)
    mu = c["avg"].double()
    for _ in range(20):   # steps with new keys that carry the mean; the window gains their centred rows
        k_new = (torch.randn((B, Hkv, d), generator=g, dtype=torch.float64) + mu).bfloat16()
        v_new = torch.randn((B, Hkv, d), generator=g).bfloat16()
        ctx.plan()
        ctx.decode(1, c["q"][:, 0].contiguous().to(DEV), k_new.to(DEV), v_new.to(DEV))
        c["win_k"] = torch.cat([c["win_k"], (k_new - c["avg"])[:, :, None]], dim=2)
        c["win_v"] = torch.cat([c["win_v"], v_new[:, :, None]], dim=2)
    got = ctx.spill_window(NL)
    sp = int(got[0])
    assert got.tolist() == [sp] * B and sp == 20
    moved_k = c["win_k"][:, :, NS:NS + sp]
    c["win_k"] = torch.cat([c["win_k"][:, :, :NS], c["win_k"][:, :, NS + sp:]], dim=2)
    c["win_v"] = torch.cat([c["win_v"][:, :, :NS], c["win_v"][:, :, NS + sp:]], dim=2)
    k_st, v_st, kn_st = (x.cpu() for x in ctx.read_cache(1))
    n2 = n + sp
    assert torch.equal(k_st[:, :, n:n2].view(torch.int16), moved_k.contiguous().view(torch.int16)), "spilled rows lost their centring"
    # the tables: the prompt's codes as built, the spilled rows' codes from the context's key hash (what the spill merged)
    spilled_codes = torch.stack([ctx.hash_keys(k_st[b, :, n:n2].contiguous().to(DEV)).cpu() for b in range(B)])
    c.update(n=n2, key=k_st[:, :, :n2].contiguous(), value=v_st[:, :, :n2].contiguous(), kn=kn_st[:, :, :n2].contiguous(),
             kcodes=torch.cat([c["kcodes"], spilled_codes], dim=-1))
    # queries near the spilled keys, so that they are sampled
    q = (moved_k[:, :, 3:4].double().repeat_interleave(c["G"], dim=1).transpose(1, 2)
         + 0.25 * torch.randn((B, 1, Hq, d), generator=g, dtype=torch.float64)).bfloat16()
    c["q"] = q
    r = run_step(ctx, c)
    check_step(c, r)
    assert all(int((r["res"][b, 0, h, : r["nnz"][b, 0, h]] >= n).sum()) > 0 for b in range(B) for h in range(Hq))


# ---- dense layers ---------------------------------------------------------------------------------------------------------
def dense_ctx(B, Hq, Hkv, M, t_max=1, impl=1, **kw):
    from magicpig_b200.ops import Context
    ctx = Context(4, 8, 2, Hq, Hkv, d, B, M, NS, NL, GEN, dense_layers=[0], alloc_dense_kv=True, device=DEV,  # (K4 L8: tables unused)
                  max_query_tokens=t_max, **kw)
    ctx.set_option("dense_impl", impl)
    ctx.set_option("out_f32", 1)
    return ctx


def run_dense(ctx, c, parents=None):
    B, T, Hq = c["q"].shape[:3]
    if T == 1:
        ctx.plan()
        out = ctx.dense_decode(0, c["q"][:, 0].contiguous().to(DEV), c["k"][:, 0].contiguous().to(DEV), c["v"][:, 0].contiguous().to(DEV))
    else:
        ctx.plan(T, parents=None if parents is None else torch.tensor(parents, dtype=torch.int32, device=DEV))
        out = ctx.dense_decode_tokens(0, T, c["q"].to(DEV), c["k"].to(DEV), c["v"].to(DEV))
    o32 = ctx.last_out_f32().cpu().reshape(B, T, Hq, d)
    assert torch.equal(out.cpu().view(torch.int16).int().reshape(B, T, Hq, d) & 0xFFFF, bf16_half_up(o32).reshape(B, T, Hq, d))
    return o32


def fill_dense(ctx, c):
    for b in range(c["B"]):
        ctx.dense_fill(0, b, c["dk"][b].to(DEV).contiguous(), c["dv"][b].to(DEV).contiguous(), c["P"])


DENSE_P = [1, 31, 32, 33, 4095, 4097, 60000]


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("P", DENSE_P)
@pytest.mark.parametrize("regime,G", [("R2", None), ("R4", None), ("R2", 16), ("R4", 16), ("R2", 32), ("R4", 32)],
                         ids=["R2", "R4", "R2-G16", "R4-G16", "R2-G32", "R4-G32"])
def test_dense_single(cuda_lib, regime, G, P, impl):
    """Single-token dense decode (dense_impl 1: GQA-shared kernel, 0: generic gather) at tile edges, and at a P whose groups
    are split over several CTAs (level-2 merge).  G = 16 / 32: more query heads per kv-head than one packed m-tile holds, on
    one m-tile or two."""
    B, Hq, Hkv = (1, 8, 1) if P > 5000 else (2, 8, 2)
    if G:
        Hq = G * Hkv
    c = make_dense(regime, B, Hq, Hkv, P, 1, seed=P + 3, place="new" if P == 1 else ("first" if P % 2 else "last"))
    o = check_dense(c)
    ctx = dense_ctx(B, Hq, Hkv, P + 256, impl=impl)
    fill_dense(ctx, c)
    assert_1e3_f32(run_dense(ctx, c).reshape(-1, d), o.reshape(-1, d))


@pytest.mark.parametrize("tree", [False, True])
@pytest.mark.parametrize("G,T", [(4, 2), (4, 4), (4, 8)], ids=["TG8", "TG16", "TG32"])
@pytest.mark.parametrize("regime", ["R2", "R4"])
def test_dense_tokens(cuda_lib, regime, G, T, tree):
    B, Hkv, P = 2, 2, 777
    parents = [TREE[:T] if T < 8 else TREE] * B if tree else None
    c = make_dense(regime, B, G * Hkv, Hkv, P, T, seed=T + 50 * tree, place="last")
    o = check_dense(c, parents)
    ctx = dense_ctx(B, G * Hkv, Hkv, P + 256, t_max=T)
    fill_dense(ctx, c)
    assert_1e3_f32(run_dense(ctx, c, parents).reshape(-1, d), o.reshape(-1, d))


@pytest.mark.parametrize("T", [1, 4])
@pytest.mark.parametrize("regime", ["R2", "R4"])
def test_dense_slots(cuda_lib, regime, T):
    """Slot mode (dense_tail_rows > 0): the sink (R2) or the large logits' prompt lives in the shared prefix; in R4 the dominant
    key is appended to request 1's tail by its first step only.  Three steps; each request against fp64 over prompt + its tail."""
    from tests.test_gpu_shared import Doc
    B, Hq, Hkv, P = 4, 8, 2, 1000
    c = make_dense(regime, B, Hq, Hkv, P, T, seed=77 + T, place="new", one_prompt=True)
    if regime == "R4":
        c["k"][[0, 2, 3], -1] = c["k"][[0, 2, 3], 0]
    hf = synth.make_hash_func(d, 4, 8, seed=1)
    ctx = dense_ctx(B, Hq, Hkv, 2048, t_max=T, num_contexts=1, dense_tail_rows=64)
    ctx.set_hash_func(hf.to(DEV))
    doc = Doc(Hkv, 600, 4, 8, hf, seed=9, P_dense=P)
    doc.dk, doc.dv = c["dk"][0].clone(), c["dv"][0].clone()
    doc.fill_store(ctx, 0)
    doc.fill_request(ctx, 0)
    for b in range(1, B):
        ctx.fork(0, b)
    assert ctx.dense_tail_rows == 64
    g = torch.Generator().manual_seed(T)
    for step in range(3):
        o = check_dense(c) if step == 0 else restate_dense(c)
        assert_1e3_f32(run_dense(ctx, c).reshape(-1, d), o.reshape(-1, d))
        # the step's rows join every request's own rows; next step: new queries, keys and values of the same kind
        c["dk"], c["dv"] = torch.cat([c["dk"], c["k"]], dim=1), torch.cat([c["dv"], c["v"]], dim=1)
        fresh = torch.randn(c["k"].shape, generator=g, dtype=torch.float64)
        c["k"] = (0.25 * fresh + c["dk"][:, :1].double()).bfloat16() if regime == "R2" else fresh.bfloat16()
        c["v"] = torch.randn(c["v"].shape, generator=g).bfloat16()
        c["q"] = (c["q"].double() * (1.0 + 0.05 * torch.randn(c["q"].shape, generator=g, dtype=torch.float64))).bfloat16()


# ---- scale invariance and option paths ------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", [1, 0])
def test_scale_invariance(cuda_lib, impl):
    """q x 2^k: SimHash normalises q and a power of two scales it exactly, so codes, nnz and index lists are bitwise those of
    q; only the outputs move (and each stays within the bar of its own fp64 restatement)."""
    c = case("R1", "last", SHAPES[0])
    base = run_step(sparse_ctx(c, impl=impl), c)
    for k in (-3, 4):
        ck = dict(c, q=(c["q"].float() * 2.0 ** k).bfloat16())
        assert torch.equal(ck["q"].float(), c["q"].float() * 2.0 ** k)
        r = run_step(sparse_ctx(ck, impl=impl), ck)
        for key in ("codes", "nnz", "res"):
            assert torch.equal(r[key], base[key]), key
        assert not torch.equal(r["o32"], base["o32"])
        check_step(ck, r)


def _same(a, b, fp32_exact=True):
    for key in ("codes", "nnz", "res"):
        assert torch.equal(a[key], b[key]), key
    if fp32_exact:
        assert torch.equal(a["o32"], b["o32"])
    else:
        assert rel_head(a["o32"], b["o32"]) <= 1e-5


@pytest.mark.parametrize("impl", [1, 0])
def test_issue_window_and_pdl(cuda_lib, impl):
    """fused_issue_win in {0, 1, 8, 32} and pdl_first in {0, 1}: bitwise the default's outputs, codes and lists."""
    c = case("R4", "last", SHAPES[2])
    base = run_step(sparse_ctx(c, impl=impl), c)
    check_step(c, base)
    for win in (0, 1, 8, 32):
        for pdl in (0, 1):
            _same(run_step(sparse_ctx(c, impl=impl, fused_issue_win=win, pdl_first=pdl), c), base)


def test_two_ctas_per_sm(cuda_lib, monkeypatch):
    """MPIG_CTA_PER_SM=2 (clusters of 512-thread CTAs): same index lists, fp32 within 1e-5, and within the bar of fp64."""
    c = case("R3", "last", SHAPES[0])
    base = run_step(sparse_ctx(c), c)
    monkeypatch.setenv("MPIG_CTA_PER_SM", "2")
    r = run_step(sparse_ctx(c), c)
    _same(r, base, fp32_exact=False)
    check_step(c, r)


def test_attend_ctas_warps(cuda_lib):
    """attend_ctas in {0, 1, 3} x attend_warps in {1, 5, 12} on the three-launch path: within 1e-5 of the default and 1e-3
    of fp64."""
    c = case("R2", "last", SHAPES[0])
    base = run_step(sparse_ctx(c, impl=0), c)
    check_step(c, base)
    for ctas in (0, 1, 3):
        for warps in (1, 5, 12):
            r = run_step(sparse_ctx(c, impl=0, attend_ctas=ctas, attend_warps=warps), c)
            _same(r, base, fp32_exact=False)
            check_step(c, r)
