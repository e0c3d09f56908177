"""The generator and fp64 restatement of chunk steps (tests/test_gpu_chunk_numerics.py, tests/test_chunk_numerics_inputs_cpu.py,
tests/test_chunk_cpu.py), and the host formula of launch_chunk_attend's key splits."""
import math

import torch

from tests.support.fp64 import BAR, centred, rel_rows

DEV = "cuda:0"
d, NS, NL, K_, L_ = 128, 4, 64, 6, 16
RD = math.sqrt(d)
CK_ROWS, CK_KT, CK_SPLIT_MAX = 128, 64, 16
P_C, N_C, GEN_C = 98000, 97932, 1100      # the chunk line: prompt, store keys (P - NS - NL), generation_buffer

PERTURBATIONS = ("sees_next_row", "misses_own_row", "window_base_off_by_one", "drop_tile_at_split_start", "drop_last_split",
                 "uncentred_chunk_keys", "no_dense_prefix", "sees_all_private", "sees_no_private", "stale_lengths")
EVERY_REQUEST = {"sees_all_private", "sees_no_private"}


# ------------------------------------------------------------------------------------------------
# host formula of launch_chunk_attend
# ------------------------------------------------------------------------------------------------
def host_splits(T, G, Hkv, B, sms, keys):
    """(m-blocks, key splits) launch_chunk_attend picks: keys = the longest request's key axis as the host sees it."""
    nmb = (T * G + CK_ROWS - 1) // CK_ROWS
    ctas = nmb * Hkv * B
    s = min(CK_SPLIT_MAX, max(1, 2 * sms // ctas)) if ctas < sms else 1
    return nmb, max(1, min(s, keys // 512))


def split_per(ntot, splits):
    """Keys per split (whole 64-key tiles) of a request whose combined key axis holds ntot keys."""
    return ((ntot + splits - 1) // splits + CK_KT - 1) // CK_KT * CK_KT


# ------------------------------------------------------------------------------------------------
# generator
# ------------------------------------------------------------------------------------------------
class Case:
    """Inputs of one chunk case for B requests on C slots (request b on slot b % C; C = B: one slot each).

    Sparse layer: per slot a centred store (Hkv, n, d) and avg (Hkv, d); per request a centred window of NS + x[b] + NL rows, of
    which the x[b] after the sinks are spilled into the slot before the chunk (spill=True).  Dense layer: per request a raw cache
    (p, Hkv, d), or with tail=True one prompt per slot (dense_tail_rows mode, the requests' tails empty).  Chunk: q (B, T, Hq, d),
    k / v (B, T, Hkv, d) raw.  Lengths are tracked as the library advances them (window / dense rows lists per request)."""

    def __init__(self, regime, B, T, Hq=32, Hkv=8, n=N_C, p=P_C, C=None, x=None, spill=False, tail=False, place="split_start",
                 sms=132, seed=0, dev=DEV, check_layers=("sparse", "dense"), splits=None):
        self.regime, self.place, self.B, self.T, self.Hq, self.Hkv, self.G = regime, place, B, T, Hq, Hkv, Hq // Hkv
        self.C = C or B
        self.n, self.p, self.tail, self.spill, self.sms, self.dev = n, p, tail, spill, sms, dev
        self.layers = check_layers
        self.fixed_splits = splits   # a captured plan's split count (the host's estimate at capture), else the exact formula
        self.x = list(x) if x is not None else [0] * B
        g = torch.Generator(device=dev).manual_seed(seed)
        self.g = g
        rnd = lambda *s: torch.randn(s, generator=g, device=dev, dtype=torch.float64)   # noqa: E731
        u = rnd(Hkv, d)
        self.u = u / u.norm(dim=-1, keepdim=True)
        self.qscale = 16.0 if regime == "R4" else 1.0
        q = 0.5 * rnd(B, T, Hq, d) + RD * self.u.repeat_interleave(self.G, 0)
        self.q = (q * self.qscale).bfloat16()
        mu = torch.zeros((Hkv, d), dtype=torch.float64, device=dev)
        if regime == "R1":   # |mu| ~ 4 |noise|, partly along the queries
            mu = 4.0 * (0.8 * rnd(Hkv, d) + 0.6 * RD * self.u)
        self.mu = mu
        self.avg = [(mu + 0.05 * rnd(Hkv, d)).bfloat16() for _ in range(self.C)]
        self.store_k = [rnd(Hkv, n, d).bfloat16() for _ in range(self.C)]
        self.store_v = [torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16() for _ in range(self.C)]
        self.win_k = [rnd(Hkv, NS + self.x[b] + NL, d).bfloat16() for b in range(B)]
        self.win_v = [torch.randn((Hkv, NS + self.x[b] + NL, d), generator=g, device=dev).bfloat16() for b in range(B)]
        ndense = self.C if tail else B
        self.dk = [(rnd(p, Hkv, d) + mu).bfloat16() for _ in range(ndense)]
        self.dv = [torch.randn((p, Hkv, d), generator=g, device=dev).bfloat16() for _ in range(ndense)]
        self.tails = [(self.dk[0][:0], self.dv[0][:0]) for _ in range(B)]   # rows past the slot prompt (tail mode)
        self.k = (rnd(B, T, Hkv, d) + mu).bfloat16()
        self.v = torch.randn((B, T, Hkv, d), generator=g, device=dev).bfloat16()
        self.priv = [[] for _ in range(self.C)]   # per slot: (request, lo, hi) spans of spilled keys, in store order
        self.vis = [[b] for b in range(B)]        # requests whose spilled keys request b sees
        self._tune()

    # -- the library's view: lengths and the combined key axis ----------------------------------------------------------------
    def slot(self, b):
        return b % self.C

    def do_spill(self, keep=NL):
        """The spill the library performs: every request's non-sink window rows but the newest `keep` go to its slot, in
        request order.  Returns the spilled counts."""
        counts = []
        for b in range(self.B):
            s, wk, wv = self.slot(b), self.win_k[b], self.win_v[b]
            m = max(wk.shape[1] - NS - keep, 0)
            lo = self.store_k[s].shape[1]
            self.store_k[s] = torch.cat([self.store_k[s], wk[:, NS:NS + m]], 1)
            self.store_v[s] = torch.cat([self.store_v[s], wv[:, NS:NS + m]], 1)
            if self.B > self.C:
                self.priv[s].append((b, lo, lo + m))
            self.win_k[b] = torch.cat([wk[:, :NS], wk[:, NS + m:]], 1)
            self.win_v[b] = torch.cat([wv[:, :NS], wv[:, NS + m:]], 1)
            counts.append(m)
        return counts

    def commit(self, kept):
        """The chunk's first kept[b] rows join request b's window and dense rows (after the step, or a rewind)."""
        for b in range(self.B):
            n = kept[b]
            self.win_k[b] = torch.cat([self.win_k[b], self.chunk_rows(b, "sparse")[0][:, :n]], 1)
            self.win_v[b] = torch.cat([self.win_v[b], self.v[b, :n].transpose(0, 1)], 1)
            rows = (self.k[b, :n], self.v[b, :n])
            if self.tail:
                self.tails[b] = (torch.cat([self.tails[b][0], rows[0]]), torch.cat([self.tails[b][1], rows[1]]))
            else:
                self.dk[b], self.dv[b] = torch.cat([self.dk[b], rows[0]]), torch.cat([self.dv[b], rows[1]])

    def chunk_rows(self, b, layer, uncentred=False):
        """(Hkv, T, d) keys and values of request b's chunk rows as layer `layer` stores them."""
        k = self.k[b].transpose(0, 1)
        if layer == "sparse" and not uncentred:
            k = centred(k, self.avg[self.slot(b)][:, None])
        return k, self.v[b].transpose(0, 1)

    def axis(self, b, layer, variant=None):
        """Request b's combined key axis: keys / values (Hkv, ntot, d), keep (ntot,) bool (private filter), nA, jb0."""
        T = self.T
        ck, cv = self.chunk_rows(b, layer, uncentred=(variant == "uncentred_chunk_keys"))
        if layer == "sparse":
            s = self.slot(b)
            ak, av = self.store_k[s], self.store_v[s]
            if variant == "stale_lengths":
                ak, av = ak[:, :self.stale_n[s]], av[:, :self.stale_n[s]]
            keep = torch.ones(ak.shape[1], dtype=torch.bool, device=self.dev)
            for r, lo, hi in self.priv[s]:
                sees = (variant == "sees_all_private") or (variant != "sees_no_private" and r in self.vis[b])
                keep[lo:hi] = sees and hi <= ak.shape[1]
            bk, bv = self.win_k[b], self.win_v[b]
        elif self.tail:
            ak, av = self.dk[self.slot(b)].transpose(0, 1), self.dv[self.slot(b)].transpose(0, 1)
            keep = torch.full((ak.shape[1],), variant != "no_dense_prefix", dtype=torch.bool, device=self.dev)
            bk, bv = self.tails[b][0].transpose(0, 1), self.tails[b][1].transpose(0, 1)
        else:
            ak = av = self.dk[b][:0].transpose(0, 1)
            keep = torch.zeros(0, dtype=torch.bool, device=self.dev)
            bk, bv = self.dk[b].transpose(0, 1), self.dv[b].transpose(0, 1)
        nA, jb0 = ak.shape[1], bk.shape[1]
        K = torch.cat([ak, bk, ck], 1)
        V = torch.cat([av, bv, cv], 1)
        keep = torch.cat([keep, torch.ones(jb0 + T, dtype=torch.bool, device=self.dev)])
        return K, V, keep, nA, jb0

    def ntot(self, b, layer):
        _, _, keep, _, _ = self.axis(b, layer)
        return keep.shape[0]

    def host_keys(self, layer):
        """The key count the host's split formula reads (exact lengths: store + window + T, or dense rows + T)."""
        if layer == "sparse":
            return max(self.store_k[self.slot(b)].shape[1] + self.win_k[b].shape[1] + self.T for b in range(self.B))
        if self.tail:
            return max(self.dk[self.slot(b)].shape[0] + self.tails[b][0].shape[0] + self.T for b in range(self.B))
        return max(self.dk[b].shape[0] + self.T for b in range(self.B))

    def splits(self, layer):
        if self.fixed_splits:
            return self.fixed_splits
        return host_splits(self.T, self.G, self.Hkv, self.B, self.sms, self.host_keys(layer))[1]

    def boundary(self, b, layer, splits=None):
        """The split boundary whose first tile drop_tile_at_split_start drops: split splits // 2 (0 with one split)."""
        sp = self.splits(layer) if splits is None else splits
        return (sp // 2) * split_per(self.ntot(b, layer), sp)

    # -- shaping the regimes ------------------------------------------------------------------------------------------------
    def _lse(self, layer, b=0):
        """Median over request b's first token's rows of the log-sum-exp of its visible scores (natural log)."""
        K, _, keep, nA, jb0 = self.axis(b, layer)
        q = self.q[b, 0].double()
        K = K[:, :nA + jb0 + 1].double()
        if layer != "sparse":   # in centred terms, as _along places keys (the dense layer's raw keys carry mu)
            K = K - self.mu[:, None]
        z = torch.einsum("hgd,hkd->hgk", q.reshape(self.Hkv, self.G, d), K) / RD
        z = z.masked_fill(~keep[None, None, :nA + jb0 + 1], -math.inf)
        return float(torch.logsumexp(z, -1).median())

    def _along(self, score, noise=0.25, count=1):
        """count keys (Hkv, count, d) along the group directions with about that score for the queries."""
        lam = score / (self.qscale * RD)
        return (noise * torch.randn((self.Hkv, count, d), generator=self.g, device=self.dev, dtype=torch.float64)
                + lam * RD * self.u[:, None]).bfloat16()

    def _set_key(self, b, layer, kidx, rows):
        """Overwrite keys [kidx, kidx + rows.shape[1]) of request b's axis (store, dense prompt or dense rows, centred / raw)."""
        if layer == "sparse":
            self.store_k[self.slot(b)][:, kidx:kidx + rows.shape[1]] = rows
        elif self.tail:
            self.dk[self.slot(b)][kidx:kidx + rows.shape[1]] = (rows.double() + self.mu[:, None]).bfloat16().transpose(0, 1)
        else:
            self.dk[b][kidx:kidx + rows.shape[1]] = (rows.double() + self.mu[:, None]).bfloat16().transpose(0, 1)

    def _in_a_or_dense(self, b, layer, k0, width):
        if layer == "sparse":
            return k0 + width <= self.store_k[self.slot(b)].shape[1]
        lo = NS + CK_KT if self.regime == "R2" else 0   # R2: not over the sinks
        return lo <= k0 and k0 + width <= (self.dk[self.slot(b)] if self.tail else self.dk[b]).shape[0]

    def _tune(self):
        B = self.B
        if self.spill:
            # each request's spilled rows lean towards the queries, so that its private keys carry mass (a request seeing none
            # of them, or everybody's, is visible); then the library's spill
            lse = self._lse("sparse")
            for b in range(B):
                xb = self.x[b]
                self.win_k[b][:, NS:NS + xb] = self._along(lse + math.log(0.6 / xb), 0.5, xb)
            self.stale_n = [self.store_k[s].shape[1] for s in range(self.C)]
            self.do_spill()
        if self.regime == "R2":
            # the sinks: the first NS window rows / dense rows along the group direction with about 3x the rest's mass, the
            # chunk's own rows as strong as one sink
            for layer in self.layers:
                lse = self._lse(layer)
                sink = self._along(lse + math.log(3.0 / NS), 0.0, NS)
                for b in range(B):
                    if layer == "sparse":
                        self.win_k[b][:, :NS] = sink
                    elif not self.tail:
                        self.dk[b][:NS] = (sink.double() + self.mu[:, None]).bfloat16().transpose(0, 1)
                if layer == "dense" and self.tail:
                    for s in range(self.C):
                        self.dk[s][:NS] = (sink.double() + self.mu[:, None]).bfloat16().transpose(0, 1)
            lse = self._lse(self.layers[0])
            own = self._along(lse + math.log(3.0 / NS), 0.25, B * self.T).double()
            self.k = (own.reshape(self.Hkv, B, self.T, d).permute(1, 2, 0, 3) + self.mu).bfloat16()
        if self.regime == "R1":
            # the window's non-sink rows (together) and each of the chunk's rows lean towards the queries with about e^-1 of the
            # context's mass, so that a token seeing one row more or less, or a spill the replay does not see, is visible even at
            # T = 1 over 98 K keys
            lse = self._lse(self.layers[0])
            for b in range(B):
                w = self.win_k[b].shape[1] - NS
                self.win_k[b][:, NS:] = self._along(lse - 1.0 - math.log(w), 1.0, w)
            own = self._along(lse - 1.0, 1.0, B * self.T).double()
            self.k = (own.reshape(self.Hkv, B, self.T, d).permute(1, 2, 0, 3) + self.mu).bfloat16()
        if self.regime == "R4":
            # the chunk's rows a little below the rest's mass each (so that a token seeing one row more or less is visible among
            # logits spread over ~18 nats); own_row: token 0's row dominates every later token
            lse = max(self._lse(layer) for layer in self.layers)
            own = self._along(lse - (0.0 if self.place == "own_row" else 1.0), 0.25, B * self.T).double()
            self.k = (own.reshape(self.Hkv, B, self.T, d).permute(1, 2, 0, 3) + self.mu).bfloat16()
            if self.place == "own_row":
                dom = self._along(lse + 3.0, 0.0, B).double()    # (Hkv, B, d)
                self.k[:, 0] = (dom.transpose(0, 1) + self.mu).bfloat16()
        # the tile at the checked split boundary carries mass (R1, R2: a share; R4: the dominant key, or a key a little below)
        for layer in self.layers:
            lse = self._lse(layer)
            for b in range(B):
                k0 = self.boundary(b, layer)
                if self.regime in ("R1", "R2") and self._in_a_or_dense(b, layer, k0, CK_KT):
                    self._set_key(b, layer, k0, self._along(lse + math.log(0.5 / CK_KT), 0.25, CK_KT))
                if self.regime == "R4":
                    start = self.place == "split_start" or (self.place == "split_end" and k0 == 0)   # one split: no split before
                    if start and self._in_a_or_dense(b, layer, k0, 1):
                        self._set_key(b, layer, k0, self._along(lse, 0.0))
                    elif self.place == "split_end" and self._in_a_or_dense(b, layer, k0 - 1, 2):
                        self._set_key(b, layer, k0 - 1, self._along(lse, 0.0))
                        self._set_key(b, layer, k0, self._along(lse - 2.0, 0.0))
                    elif self.place == "own_row" and self._in_a_or_dense(b, layer, k0, 1):
                        self._set_key(b, layer, k0, self._along(lse - 2.0, 0.0))

    # -- restatement ----------------------------------------------------------------------------------------------------------
    def perturbations(self, layer, capture=False):
        names = ["misses_own_row", "drop_tile_at_split_start"]
        if self.T > 1:   # (at T = 1 there is no next row, and a base one row late differs only by the first window row)
            names += ["sees_next_row", "window_base_off_by_one"]
        sp = self.splits(layer)
        if sp > 1 and any((sp - 1) * split_per(self.ntot(b, layer), sp) < self.ntot(b, layer) for b in range(self.B)):
            names.append("drop_last_split")   # (not when every request's last split is empty)
        if self.regime == "R1" and layer == "sparse":
            names.append("uncentred_chunk_keys")
        if layer == "dense" and self.tail:
            names.append("no_dense_prefix")
        if layer == "sparse" and self.B > self.C and any(self.priv):
            names += ["sees_all_private", "sees_no_private"]
        if capture and layer == "sparse":
            names.append("stale_lengths")
        return names

    def restate(self, layer, variant=None, splits=None, block=1 << 26):
        """fp64 output (B, T, Hq, d) of the chunk step on `layer` ("sparse" / "dense") under an optional perturbation."""
        B, T, G = self.B, self.T, self.G
        o = torch.empty((B, T, self.Hq, d), dtype=torch.float64, device=self.dev)
        sp = self.splits(layer) if splits is None else splits
        for b in range(B):
            K, V, keep, nA, jb0 = self.axis(b, layer, variant)
            n = K.shape[1]
            lim = nA + jb0 + torch.arange(T, device=self.dev)
            if variant in ("sees_next_row", "window_base_off_by_one"):
                lim = lim + 1
            if variant == "misses_own_row":
                lim = lim - 1
            if variant == "window_base_off_by_one":   # range B read from its second row: one row lost, one row too many
                keep = keep.clone()
                keep[nA] = False
            if variant == "drop_tile_at_split_start":
                keep = keep.clone()
                k0 = self.boundary(b, layer, sp)
                keep[k0:k0 + CK_KT] = False
            if variant == "drop_last_split":
                keep = keep.clone()
                keep[(sp - 1) * split_per(n, sp):] = False
            rows = max(1, block // max(n, 1))
            lim_r = lim.repeat_interleave(G)
            ar = torch.arange(n, device=self.dev)
            for h in range(self.Hkv):
                q = self.q[b, :, h * G:(h + 1) * G].reshape(T * G, d).double()
                Kh, Vh = K[h].double(), V[h].double()
                out = torch.empty((T * G, d), dtype=torch.float64, device=self.dev)
                for r0 in range(0, T * G, rows):
                    z = (q[r0:r0 + rows] @ Kh.t()) / RD
                    vis = (ar[None] <= lim_r[r0:r0 + rows, None]) & keep[None]
                    z = z.masked_fill(~vis, -math.inf)
                    out[r0:r0 + rows] = torch.softmax(z, -1) @ Vh
                o[b, :, h * G:(h + 1) * G] = out.reshape(T, G, d)
        return o

    def check_inputs(self, layer, capture=False):
        """Before any library call: every named perturbation moves some row (every request: EVERY_REQUEST) by >= 10x the bar.
        Returns the restatement and {perturbation: how far it moves the output}."""
        o = self.restate(layer)
        assert bool(torch.isfinite(o).all())
        moved = {}
        for name in self.perturbations(layer, capture):
            a = self.restate(layer, name)
            per_req = [rel_rows(a[b], o[b]) for b in range(self.B)]
            moved[name] = min(per_req) if name in EVERY_REQUEST else max(per_req)
            assert moved[name] >= 10 * BAR, f"{self.regime} {layer}: '{name}' moves the output by {moved[name]:.2e} only"
        return o, moved
