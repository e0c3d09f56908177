"""The long-generation lines' state on the host: the generation schedule (T-token steps with per-request rewinds, chunk steps,
a spill whenever a window is full), the dense layer's prompt and per-request tails in shared-prefix mode, the fp64 restatements
of dense steps and chunks over those tails with their named perturbations, and dense_partition_of's work items restated in
Python.  Pure torch on whichever device holds the tensors; nothing here calls the library."""
import math

import torch

from tests.support.fp64 import BAR, causal_ref, rel_rows, softmax_state, unit, visible
from tests.support.library import NS, d

RD = math.sqrt(d)
TILE = 32                 # rows per tile of the dense kernel (attend_common.cuh)
A_DOM = 1.5               # the dominant tail row: A_DOM * sqrt(d) * u; other tail rows ~ 0.25 N(0, 1) + sqrt(d) * u
A_STEP = {"R2": 1.3, "R4": 1.0}   # the check step's own keys along u (R2: strong enough that dropping the newest row shows)


# ------------------------------------------------------------------------------------------------
# the schedule
# ------------------------------------------------------------------------------------------------
def schedule(targets, T, w0, wcap, keep, chunk_at=(), t_chunk=0):
    """Events that take every request b from a window of w0 rows and an empty tail to targets[b] committed tokens:
      ("spill", g): spill_window(keep) moves g[b] rows of request b (issued whenever the next step does not fit the fullest window);
      ("step", drops): plan(T), a T-token step, rewind(drops);
      ("chunk", drops): plan_chunk(t_chunk), a chunk step, rewind(drops) -- once request 0 has committed chunk_at[i] tokens.
    The request with the largest target drops least, so that its window is the fullest at most spills; the others drop 0 or 1
    rows of each step in a rotating pattern.  A request that has reached its target drops the whole step."""
    B = len(targets)
    top = max(range(B), key=lambda b: targets[b])
    done, w, ev, s, chunks = [0] * B, [w0] * B, [], 0, list(chunk_at)

    def fit(n):
        if max(w) + n > wcap:
            ev.append(("spill", [max(0, x - NS - keep) for x in w]))
            for b in range(B):
                w[b] = min(w[b], NS + keep)

    def run(kind, n, drop):
        drops = [min(n, max(drop(b), n - (targets[b] - done[b]))) for b in range(B)]
        ev.append((kind, drops))
        for b in range(B):
            done[b] += n - drops[b]
            w[b] += n - drops[b]

    while any(done[b] < targets[b] for b in range(B)):
        if chunks and done[0] >= chunks[0]:
            chunks.pop(0)
            fit(t_chunk)
            run("chunk", t_chunk, lambda b: (b * 5) % 7)
            continue
        fit(T)
        run("step", T, lambda b: int(s % 5 == 0) if b == top else (s * 7 + b * 3) % 4 // 2)
        s += 1
    return ev, w


# ------------------------------------------------------------------------------------------------
# the dense layer: one prompt, per-request tails
# ------------------------------------------------------------------------------------------------
class DenseTails:
    """Host mirror of a dense layer in shared-prefix mode.  The prompt dk / dv (P, Hkv, d) is N(0, 1); every row a request
    commits after it lies along the kv-group's direction u (0.25 N(0, 1) + sqrt(d) u), so that queries along u put most of their
    mass on the tails; request b's tail row dom_at[b] is the dominant row A_DOM sqrt(d) u."""

    def __init__(self, B, P, R, Hkv, dom_at, seed, dev):
        self.g = torch.Generator(device=dev).manual_seed(seed)
        self.B, self.P, self.R, self.Hkv, self.dev, self.dom_at = B, P, R, Hkv, dev, list(dom_at)
        self.u = unit(self.rnd, Hkv)
        self.dk = self.rnd(P, Hkv, d).bfloat16()
        self.dv = torch.randn((P, Hkv, d), generator=self.g, device=dev).bfloat16()
        self.tk = torch.zeros((B, R, Hkv, d), dtype=torch.bfloat16, device=dev)
        self.tv = torch.zeros_like(self.tk)
        self.tl = [0] * B

    def rnd(self, *s):
        return torch.randn(s, generator=self.g, device=self.dev, dtype=torch.float64)

    def step_rows(self, T, keep):
        """k / v (B, T, Hkv, d) of a generation step; of request b's rows the first keep[b] are committed, and the one that lands
        on tail row dom_at[b] is the dominant row."""
        k = (0.25 * self.rnd(self.B, T, self.Hkv, d) + RD * self.u).bfloat16()
        v = torch.randn((self.B, T, self.Hkv, d), generator=self.g, device=self.dev).bfloat16()
        for b in range(self.B):
            j = self.dom_at[b] - self.tl[b]
            if 0 <= j < keep[b]:
                k[b, j] = (A_DOM * RD * self.u).bfloat16()
        return k, v

    def commit(self, k, v, keep):
        for b in range(self.B):
            n, i = keep[b], self.tl[b]
            assert i + n <= self.R, f"request {b}: tail past {self.R} rows"
            self.tk[b, i:i + n], self.tv[b, i:i + n] = k[b, :n], v[b, :n]
            self.tl[b] += n

    def fork(self, src, dst):
        self.tk[dst], self.tv[dst], self.tl[dst] = self.tk[src].clone(), self.tv[src].clone(), self.tl[src]

    def check_step(self, regime, T, Hq):
        """q (B, T, Hq, d) and k / v (B, T, Hkv, d) of a check step: queries along u (R4: x 16), keys along u."""
        G = Hq // self.Hkv
        q = 0.5 * self.rnd(self.B, T, Hq, d) + RD * self.u.repeat_interleave(G, 0)
        if regime == "R4":
            q = q * 16.0
        k = (0.25 * self.rnd(self.B, T, self.Hkv, d) + A_STEP[regime] * RD * self.u).bfloat16()
        v = torch.randn((self.B, T, self.Hkv, d), generator=self.g, device=self.dev).bfloat16()
        return q.bfloat16(), k, v


def chunk_size(T, G):
    """Requests of one slot per chunk of the dense kernel in shared-prefix mode (launch_attend_dense: max(1, 32 / (T G)))."""
    return max(1, 32 // (T * G))


def _tail_of(dt, b, variant, cm):
    """The tail rows request b's query rows see (k, v (n, Hkv, d)), under a named perturbation."""
    src = 0 if variant == "tail_of_request_0" else b
    k, v = dt.tk[src, :dt.tl[src]], dt.tv[src, :dt.tl[src]]
    if variant == "sees_previous_member_tail" and b % cm:
        p = b - 1   # the member before b in its chunk: its tail lies before b's in the group's rows
        k, v = torch.cat([dt.tk[p, :dt.tl[p]], k]), torch.cat([dt.tv[p, :dt.tl[p]], v])
    if variant == "drop_tail_tile":   # the 32-row tile around the dominant row, in the middle of the tail
        t0 = TILE * (dt.dom_at[b] // TILE)
        k, v = torch.cat([k[:t0], k[t0 + TILE:]]), torch.cat([v[:t0], v[t0 + TILE:]])
    return k, v


def restate_tails(dt, q, k, v, parents=None, variant=None):
    """fp64 output (B, T, Hq, d) of a dense step over the prompt, request b's own tail and the step's rows visible to token t
    (causal, or its ancestors in a tree).  variant: tail_of_request_0, sees_previous_member_tail (needs chunks of >= 2
    members), drop_tail_tile, drop_newest (token t does not see its own row), skip_rescale (row-granular, as restate_dense)."""
    B, T, Hq = q.shape[:3]
    G = Hq // dt.Hkv
    cm = chunk_size(T, G)
    o = torch.zeros((B, T, Hq, d), dtype=torch.float64, device=q.device)
    for b in range(B):
        tk, tv = _tail_of(dt, b, variant, cm)
        n0 = dt.P + tk.shape[0]
        mask = torch.zeros((n0 + T, T), dtype=torch.bool, device=q.device)
        mask[:n0] = True
        for t in range(T):
            rows = visible(parents, b, t) + ([] if variant == "drop_newest" else [t])
            mask[[n0 + j for j in rows], t] = True
        mask = mask.repeat_interleave(G, 1)                                   # (rows, T*G): column t*G + j
        for g in range(dt.Hkv):
            kk = torch.cat([dt.dk[:, g], tk[:, g], k[b, :, g]]).double()
            vv = torch.cat([dt.dv[:, g], tv[:, g], v[b, :, g]]).double()
            Q = q[b, :, g * G:(g + 1) * G].double().reshape(T * G, d)
            z = ((kk @ Q.t()) / RD).masked_fill(~mask, -math.inf)
            if variant == "skip_rescale":
                for c in range(T * G):
                    o[b, c // G, g * G + c % G], _ = softmax_state(z[:, c], vv, True, tile=1)
            else:
                o[b, :, g * G:(g + 1) * G] = (torch.softmax(z, 0).t() @ vv).reshape(T, G, d)
    return o


def tail_share(dt, q):
    """The smallest share of the softmax mass that the tails take, over every request's query rows (single-token queries)."""
    B, T, Hq = q.shape[:3]
    G = Hq // dt.Hkv
    worst = 1.0
    for b in range(B):
        for g in range(dt.Hkv):
            Q = q[b, :, g * G:(g + 1) * G].double().reshape(-1, d)
            zp = torch.logsumexp(dt.dk[:, g].double() @ Q.t() / RD, 0)
            zt = torch.logsumexp(dt.tk[b, :dt.tl[b], g].double() @ Q.t() / RD, 0)
            worst = min(worst, float(torch.sigmoid(zt - zp).min()))
    return worst


def score_span(dt, q):
    """The smallest span (max - min, nats) of a query row's scores over the prompt and its tail."""
    B, T, Hq = q.shape[:3]
    G = Hq // dt.Hkv
    span = math.inf
    for b in range(B):
        for g in range(dt.Hkv):
            Q = q[b, :, g * G:(g + 1) * G].double().reshape(-1, d)
            z = torch.cat([dt.dk[:, g], dt.tk[b, :dt.tl[b], g]]).double() @ Q.t() / RD
            span = min(span, float((z.max(0).values - z.min(0).values).min()))
    return span


def dense_perturbations(regime, T, G):
    names = ["drop_newest" if regime == "R2" else "skip_rescale", "tail_of_request_0", "drop_tail_tile"]
    if chunk_size(T, G) > 1:
        names.append("sees_previous_member_tail")
    return names


def check_dense_tails(dt, regime, q, k, v, parents=None):
    """Before any library call: the regime's property holds (R2: the tails take >= 90 % of every query row's mass over the
    prompt and its tail; R4: scores span >= 40 nats) and every named perturbation moves the fp64 output by >= 10x the bar.
    Returns (o, {perturbation: how far it moves the output})."""
    if regime == "R2":
        share = tail_share(dt, q)
        assert share >= 0.9, f"R2: the tails take {share:.3f} of the mass only"
    else:
        span = score_span(dt, q)
        assert span >= 40.0, f"R4: scores span {span:.1f} nats only"
    o = restate_tails(dt, q, k, v, parents)
    moved = {}
    for name in dense_perturbations(regime, q.shape[1], q.shape[2] // dt.Hkv):
        moved[name] = rel_rows(restate_tails(dt, q, k, v, parents, name), o)
        assert moved[name] >= 10 * BAR, f"dense {regime}: '{name}' moves the output by {moved[name]:.2e} only"
    return o, moved


def restate_chunk(dt, q, k, v, variant=None):
    """fp64 output (B, T, Hq, d) of a dense chunk step: token t of request b attends to the prompt, b's tail before the chunk
    and the chunk's rows [0, t].  variant "ignores_tail": the tail before the chunk is left out."""
    B, T, Hq = q.shape[:3]
    G = Hq // dt.Hkv
    o = torch.zeros((B, T, Hq, d), dtype=torch.float64, device=q.device)
    for b in range(B):
        n = 0 if variant == "ignores_tail" else dt.tl[b]
        for g in range(dt.Hkv):
            kctx = torch.cat([dt.dk[:, g], dt.tk[b, :n, g]])
            vctx = torch.cat([dt.dv[:, g], dt.tv[b, :n, g]])
            o[b, :, g * G:(g + 1) * G] = causal_ref(q[b, :, g * G:(g + 1) * G], kctx, vctx, k[b, :, g], v[b, :, g])
    return o


# ------------------------------------------------------------------------------------------------
# dense_partition_of in Python
# ------------------------------------------------------------------------------------------------
def dense_items(rows, nw):
    """Work items (group, r_lo, r_hi) of attend_dense_kernel's partition of groups with rows[g] rows over nw warps."""
    NG, total = len(rows), sum(rows)
    Rp = max(TILE, -(-total // (nw - NG))) if nw > NG else 0x3fffffff
    items = []
    for g, t in enumerate(rows):
        w = max(1, t // Rp) if t > 0 else 0
        if w == 0:
            continue
        c = -(-t // w)
        items += [(g, p * c, min(p * c + c, t)) for p in range(w)]
    return items


def tail_items(P, tails, T, G, Hkv, nw):
    """In shared-prefix mode with every request bound to one slot whose prompt has P rows and request b's tail tails[b] rows
    (the step's T rows included): (items wholly inside one member's tail, items that start strictly inside a member's tail)."""
    cm = chunk_size(T, G)
    B = len(tails)
    chunks = [list(range(c, min(c + cm, B))) for c in range(0, B, cm)]
    rows, spans = [], []
    for ch in chunks:
        pc, sp = P, []
        for b in ch:
            sp.append((pc, pc + tails[b]))
            pc += tails[b]
        for _ in range(Hkv):
            rows.append(pc)
            spans.append(sp)
    inside = boundary = 0
    for g, lo, hi in dense_items(rows, nw):
        for a, e in spans[g]:
            inside += int(a <= lo and hi <= e and hi > lo)
            boundary += int(a < lo < e)
    return inside, boundary


# ------------------------------------------------------------------------------------------------
# the sparse layer's private keys after shared spills
# ------------------------------------------------------------------------------------------------
class PrivateRuns:
    """Host model of one slot's private keys: the prompt has n keys; spill i appends request 0's g[0] rows, then request 1's, ...
    Each request sees its own runs (and, after a fork, the runs of the request it continues)."""

    def __init__(self, B, n):
        self.B, self.n, self.total = B, n, n
        self.runs = [[] for _ in range(B)]   # per request its runs (lo, hi), absolute store offsets, in spill order

    def spill(self, g):
        out = []
        for b in range(self.B):
            lo = self.total
            self.total += g[b]
            if g[b]:
                self.runs[b].append((lo, self.total))
            out.append((lo, self.total))
        return out

    def fork(self, src, dst):
        self.runs[dst] = list(self.runs[src])

    def masks(self, runs_of, dev):
        out = []
        for b in range(self.B):
            m = torch.zeros(self.total, dtype=torch.bool, device=dev)
            m[:self.n] = True
            for lo, hi in runs_of[b]:
                m[lo:hi] = True
            out.append(m)
        return out

    def visibility(self, M, dev):
        """The expected visibility words of the slot, int32 (M,): bit b of word p = request b sees private key n + p."""
        v = torch.zeros(M, dtype=torch.int64, device=dev)
        for b in range(self.B):
            for lo, hi in self.runs[b]:
                v[lo - self.n:hi - self.n] |= 1 << b
        return v.int()
