"""The fp64 side of the numerics tests: the 1e-3 bar and its metric, bf16 roundings, the fp64 restatement of the sparse decode
step, SimHash codes in fp64, the causal reference of chunk steps and the C oracle's decode chain.  Pure torch / numpy and the
CPU oracle: nothing here touches the library or a GPU unless handed tensors that live there."""
import math

import numpy as np
import torch

import oracle

d = 128
BAR = 1e-3
TILE = 16                      # rows per tile of the restatement's online softmax (the sparse kernels' tile)
# SimHash parity: exact bf16 products, fp32 accumulation in a different order than the oracle's fp64 -- a code may differ from
# the oracle's only where one of its K projections is within accumulation noise of zero.  eps is relative to the projection's
# own scale (its standard deviation: |norm_q| = 1 and N(0,1) hash entries give 1.0 for queries; keys are not normalised).
SIMHASH_EPS = 2e-5


# ------------------------------------------------------------------------------------------------
# bf16 roundings
# ------------------------------------------------------------------------------------------------
def bf16_half_up(x: torch.Tensor) -> torch.Tensor:
    """The ABI's fp32 -> bf16 rounding (add 2^15, truncate), as bit patterns."""
    u = x.float().cpu().numpy().view(np.uint32).astype(np.uint64)
    return torch.from_numpy((((u + 0x8000) >> 16) & 0xFFFF).astype(np.int32))


def bf16_rne(x: torch.Tensor) -> torch.Tensor:
    """fp64 -> the nearest bf16 value (ties to even), as fp64, in ONE rounding (no detour through fp32).  bf16 keeps 8
    significant bits; its subnormals are spaced 2^-133."""
    x = x.double()
    _, e = torch.frexp(x)
    ulp = torch.ldexp(torch.ones_like(x), (e - 8).clamp(min=-133))
    return torch.round(x / ulp) * ulp      # torch.round: half to even


def bf16_from_u16(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16)


# ------------------------------------------------------------------------------------------------
# the bar
# ------------------------------------------------------------------------------------------------
def rel_rows(a: torch.Tensor, o: torch.Tensor) -> float:
    """max over rows (the last axis: a head's or a token's output) of max|a - o| / max|o|: the bar's metric."""
    n = a.shape[-1]
    a, o = a.double().reshape(-1, n), o.double().to(a.device).reshape(-1, n)
    return float(((a - o).abs().amax(-1) / o.abs().amax(-1).clamp_min(1e-30)).max())


def rel_max(a: torch.Tensor, b: torch.Tensor) -> float:
    """max|a - b| / max|b| over the whole tensors (two runs of the library against each other)."""
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def assert_1e3_f32(out_f32: torch.Tensor, o_exact: torch.Tensor, tol: float = BAR):
    """The product path's fp32 output (option "out_f32": the value BEFORE the ABI's bf16 rounding) against the oracle's
    un-rounded result, per head: max|diff| <= tol * max|o|  (BASELINE.json: "within 1e-3 relative on the attention output")."""
    worst = rel_rows(out_f32, o_exact)
    assert worst <= tol, f"fp32 output differs from the oracle by {worst:.3e} relative (bar {tol:g})"


def assert_1e3_before_rounding(out_bf16: torch.Tensor, o_exact: torch.Tensor, tol: float = BAR):
    """out is the bf16 the ABI prescribes; o_exact the same quantity before that rounding.  Error budget per element:
    half a bf16 ulp of o_exact (<= |o| * 2^-8, round-to-nearest) + tol * max|o| for the arithmetic."""
    o = o_exact.double()
    diff = (out_bf16.double() - o).abs()
    bound = o.abs() * 2.0 ** -8 + tol * o.abs().max()
    worst = float((diff - bound).max())
    assert worst <= 0.0, f"arithmetic error beyond {tol:g} relative before the bf16 rounding (excess {worst:.3e})"


def assert_rounded_half_up(out_bf16: torch.Tensor, out_f32: torch.Tensor, label: str = "output"):
    """The bf16 output is the fp32 output rounded once, half-up, element for element."""
    got = out_bf16.detach().cpu().reshape(-1).view(torch.int16).int() & 0xFFFF
    want = bf16_half_up(out_f32).reshape(-1)
    assert got.shape == want.shape, f"{label}: {got.numel()} bf16 elements, {want.numel()} fp32 elements"
    ulps = (got - want).abs()
    assert not bool(ulps.any()), (f"{label}: {int((ulps > 0).sum())} bf16 elements are not the fp32 output rounded half-up, "
                                  f"up to {int(ulps.max())} ulp off")


# ------------------------------------------------------------------------------------------------
# the sparse decode step in fp64
# ------------------------------------------------------------------------------------------------
def unit(rnd, *shape):
    """Unit vectors (*shape, d) from the fp64 normal draw rnd(*shape, d)."""
    u = rnd(*shape, d)
    return u / u.norm(dim=-1, keepdim=True)


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


def visible(parents, b, t):
    """Earlier step tokens token t attends to besides itself: all before it (chain) or its ancestors (tree)."""
    if parents is None:
        return list(range(t))
    anc, j = [], parents[b][t]
    while j >= 0:
        anc.append(j)
        j = parents[b][j]
    return anc[::-1]


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


# A sparse case c holds, per context slot s, c["slots"][s] = dict(key / value (Hkv, n, d) centred store, kn (Hkv, n), avg
# (Hkv, d), kcodes (Hkv, L, n)); request b reads slot c["slot_of"][b] and its own window c["win_k"][b] / c["win_v"][b]
# (Hkv, w_b, d, centred); c["vis"]: None, or per request a bool mask of the slot's keys it sees (after a shared spill).
def sample_sets(c, codes, wrong=False):
    """Index lists (ascending) of the keys of request b's slot (the next slot: wrong) that collide with its query codes in >= 2
    tables, restricted to the keys it sees (c["vis"]): codes int32 (B, T, Hq, L) -> [b][t][h] LongTensor."""
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


def avg_of(c, b):
    return c["slots"][c["slot_of"][b]]["avg"]


def head_mask(c, heads):
    return torch.ones((c["B"], c["Hq"]), dtype=torch.bool) if heads is None else heads


def _window(c, b, t, g, variant=None, parents=None):
    """Request b's window rows for token t of group g: its filled rows, the step's visible rows and the token, centred."""
    wb = 0 if variant == "window_of_request_0" else b
    new = c["k_new"][b, :, g] if variant == "uncentred" else c["k_new"][b, :, g] - avg_of(c, b)[g]
    vis = visible(None if variant == "tree_as_chain" else parents, b, t)
    wk = torch.cat([c["win_k"][wb][g], new[vis], new[t:t + 1]])
    wv = torch.cat([c["win_v"][wb][g], c["v_new"][b, vis, g], c["v_new"][b, t:t + 1, g]])
    if variant == "drop_newest":
        wk, wv = wk[:-1], wv[:-1]
    return wk, wv


def restate(c, codes, variant=None, parents=None, heads=None, sets=None):
    """fp64 restatement of the sparse decode step of case c over each request's slot store and own window.  The sample set
    comes from collision counts over `codes` (B, T, Hq, L) unless `sets` is given; cos is clamped to [-1, 1], the LSH weight
    applied, the window rows plus bf16(k_new - avg) attended under the causal / ancestor mask of the step, and the two halves
    merged by their base-2 LSEs.  Returns (o (B, T, Hq, d), lse_s (B, T, Hq) the sampled half's base-2 LSE, share (B, T, Hq)
    the window's share of the merged mass).  variant: a named perturbation (uncentred, drop_newest, ln_merge, skip_rescale,
    drop_sampled, window_of_request_0, window_of_head_0, wrong_document, tree_as_chain: the ancestor mask read as a chain) or
    None.  heads: bool (B, Hq), the heads to restate
    (None: all)."""
    B, T, Hq = c["q"].shape[:3]
    G, K, L = c["G"], c["K"], c["L"]
    wrong = variant == "wrong_document"
    if sets is None:
        sets = sample_sets(c, codes, wrong)
    hm = head_mask(c, heads)
    o = torch.zeros((B, T, Hq, d), dtype=torch.float64, device=c["q"].device)
    lse_s = torch.full((B, T, Hq), -math.inf, dtype=torch.float64)
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
                    zw = (wk.double() @ qw.double()) / math.sqrt(d)
                    if variant == "skip_rescale":
                        o[b, t, h], _ = softmax_state(torch.cat([zw, zs]), torch.cat([wv, st["value"][g, idx]]), True)
                        continue
                    o_s, l_s = softmax_state(zs, st["value"][g, idx])
                    o_w, l_w = softmax_state(zw, wv)
                    lse_s[b, t, h] = l_s
                    if variant == "drop_sampled":
                        o[b, t, h] = o_w
                        continue
                    o[b, t, h] = merge2(o_w, l_w, o_s, l_s, natural=(variant == "ln_merge"))
                    share[b, t, h] = 1.0 / (1.0 + 2.0 ** (l_s - l_w)) if l_s > -math.inf else 1.0
    return o, lse_s, share


# ------------------------------------------------------------------------------------------------
# chunk steps and the C oracle's decode chain
# ------------------------------------------------------------------------------------------------
def centred(k, avg):
    """bf16(k - avg) with an fp32 subtraction, as the append kernel centres a sparse layer's keys."""
    return (k.float() - avg.float()).bfloat16()


def causal_ref(q, kctx, vctx, kc, vc):
    """Exact softmax attention of one kv-group's chunk in fp64.  q (T, G, d) queries of the chunk's T tokens; kctx / vctx (n, d)
    rows every token sees; kc / vc (T, d) the chunk's own rows, token t seeing rows [0, t].  Scale 1/sqrt(d).  -> (T, G, d) fp64."""
    T, G, d = q.shape
    K = torch.cat([kctx.double(), kc.double()], 0)
    V = torch.cat([vctx.double(), vc.double()], 0)
    n = kctx.shape[0]
    s = torch.einsum("tgd,kd->tgk", q.double(), K) / d ** 0.5
    j = torch.arange(T, device=q.device)
    mask = torch.ones((T, n + T), dtype=torch.bool, device=q.device)
    mask[:, n:] = j[None, :] <= j[:, None]
    s = s.masked_fill(~mask[:, None, :], float("-inf"))
    return torch.einsum("tgk,kd->tgd", torch.softmax(s, dim=-1), V)


def oracle_decode(t, q, k_new, v_new, win_k, win_v, G):
    """Reference semantics of attnserver.py:261-312 on the CPU oracle, for one layer.
    Returns (o, nnz, codes, o_exact): o follows the reference's data flow (the CPU operator rounds its output to bf16 before
    merge_state); o_exact is the same quantity with NO intermediate rounding -- the oracle's fp32 probabilities times V in
    fp64, merged with the window state in fp64 -- i.e. what the 1e-3 bar is measured against."""
    B, Hq, Hkv, d, K, L, n, M = t["B"], t["Hq"], t["Hkv"], t["d"], t["K"], t["L"], t["n"], t["M"]
    H = B * Hq
    codes, _ = oracle.simhash(q.reshape(H, d), t["hash_func"], K, L)
    sc, si = t["kcodes"].sort()
    res, nz = [], []
    for b in range(B):
        T = oracle.Tables(Hkv, L, K, M)
        T.fill(sc[b].contiguous(), si[b].int().contiguous())
        r, n_, _ = oracle.batch_retrieve(T, codes[b * Hq:(b + 1) * Hq].contiguous(), G)
        res.append(r), nz.append(n_)
    res, nz = torch.cat(res), torch.cat(nz)
    kp = torch.zeros((B * Hkv, M, d), dtype=torch.bfloat16); vp = torch.zeros((B * Hkv, M, d), dtype=torch.bfloat16); knp = torch.zeros((B * Hkv, M))
    kp[:, :n], vp[:, :n], knp[:, :n] = t["key"].reshape(-1, n, d), t["value"].reshape(-1, n, d), t["key_norm"].reshape(-1, n)
    qn = q.reshape(H, d).float().norm(p=2, dim=-1)
    o_s, mve, score = oracle.attention_wrapper(kp, vp, knp, K, L, q.reshape(H, d), qn, res, nz, want_score=True)
    # window = stored window rows + the new (centred) key/value (attnserver.py:275-296)
    kc = (k_new.reshape(B * Hkv, 1, d) - t["avg_k"].reshape(B * Hkv, 1, d))
    wk = torch.cat([win_k.reshape(B * Hkv, -1, d), kc], dim=1)
    wv = torch.cat([win_v.reshape(B * Hkv, -1, d), v_new.reshape(B * Hkv, 1, d)], dim=1)
    o_w, lse_w = oracle.window_attention(wk, wv, q.reshape(H, d), G)
    o, lse = oracle.merge_state(o_w, lse_w, o_s.float(), mve[1])
    # un-rounded: sum_j p_j V_j in fp64, LSE merge in fp64
    o_s64 = torch.zeros((H, d), dtype=torch.float64)
    for h in range(H):
        sel = res[h, : nz[h]].long()
        if len(sel):
            o_s64[h] = score[h, : nz[h]].double() @ vp[h // G][sel].double()
    lw, ls = lse_w.double(), mve[1].double()
    m = torch.maximum(lw, ls)
    a, b_ = torch.exp2(lw - m), torch.exp2(ls - m)          # ls = -inf (nnz = 0) -> b_ = 0
    o_exact = (a[:, None] * o_w.double() + b_[:, None] * o_s64) / (a + b_)[:, None]
    return o, nz, codes, o_exact
