"""The generator and fp64 restatement of prefill attention (tests/test_gpu_prefill.py, tests/test_prefill_cpu.py): causal GQA
attention of q (q_len, Hq, d) over k / v (kv_len, Hkv, d), query i seeing keys [0, kv_len - q_len + i], under the named
perturbations a kernel bug would amount to.  Pure torch: runs wherever the tensors live."""
import math

import torch
import torch.nn.functional as F

from tests.support.fp64 import BAR, rel_rows

d = 128
RD = math.sqrt(d)
PF_BM, PF_KT = 128, 128      # query rows per m-block, keys per tile (csrc/attend_prefill.cu)
REGIMES = ("mean", "sinks", "sharp")
NS = 4                       # the sink keys of the "sinks" regime
PERTURBATIONS = ("limit_plus_1", "limit_minus_1", "top_left", "head_mod", "drop_last_tile", "skip_rescale")


def tokens_per_block(G):
    """Query tokens of one m-block: floor(128 / G), so a block's rows t*G + g never split a token."""
    return PF_BM // G


def check_rows(q_len, G, n_random=1024, seed=0):
    """The query tokens a long case is checked on: the first and last, each m-block's first and last, and n_random more."""
    tb = tokens_per_block(G)
    starts = torch.arange(0, q_len, tb)
    rows = torch.cat([torch.tensor([0, q_len - 1]), starts, (starts + tb - 1).clamp(max=q_len - 1),
                      torch.randint(0, q_len, (n_random,), generator=torch.Generator().manual_seed(seed))])
    return torch.unique(rows)


class Case:
    """q (q_len, Hq, d), k / v (kv_len, Hkv, d) bf16 on `dev`, shaped for one regime:
      mean   keys with a large common mean (|mu| ~ 4 |noise|, partly along the queries: large common score offsets);
      sinks  the first NS keys along the queries with about 3x the mass of the rest (attention sinks);
      sharp  queries at 16x scale (a few keys take the probability) and one dominant key on a key-tile edge.
    Wherever the chunk has context (q_len < kv_len) the chunk's own keys each lean towards the queries with a little less than the
    context's mass, so that a row seeing one key more or less is visible; the first key of the second tile raises the running
    max, and the last key carries about half of the last row's mass."""

    def __init__(self, regime, q_len, kv_len, Hq=32, Hkv=8, seed=0, dev="cuda:0"):
        assert regime in REGIMES and 1 <= q_len <= kv_len
        self.regime, self.q_len, self.kv_len, self.Hq, self.Hkv, self.G = regime, q_len, kv_len, Hq, Hkv, Hq // Hkv
        self.off, self.dev = kv_len - q_len, dev
        g = torch.Generator(device=dev).manual_seed(seed)
        self.g = g
        rnd = lambda *s: torch.randn(s, generator=g, device=dev, dtype=torch.float64)   # noqa: E731
        u = rnd(Hkv, d)
        self.u = u / u.norm(dim=-1, keepdim=True)
        self.qscale = 16.0 if regime == "sharp" else 1.0
        q = 0.5 * rnd(q_len, Hq, d) + RD * self.u.repeat_interleave(self.G, 0)[None]
        self.q = (q * self.qscale).bfloat16()
        k = rnd(kv_len, Hkv, d)
        if regime == "mean":
            k = k + 4.0 * (0.8 * rnd(Hkv, d) + 0.6 * RD * self.u)[None]
        self.k = k.bfloat16()
        self.v = torch.randn((kv_len, Hkv, d), generator=g, device=dev).bfloat16()
        if regime == "sinks" and kv_len > NS:
            self.k[:NS] = self._along(self._lse(NS + 1, kv_len) + math.log(3.0 / NS), 0.0, NS)
        edge = kv_len
        if regime == "sharp":   # the last key of a tile, inside the context when it holds one: planted before the chunk's keys
            span = self.off if self.off >= PF_KT else kv_len
            edge = min(kv_len - 1, PF_KT * max(1, span // (2 * PF_KT)) - 1)
            if edge < self.off:
                self.k[edge:edge + 1] = self._along(self._lse(0, kv_len) + 3.0, 0.0, 1)
        if self.off > 0:
            self.k[self.off:] = self._along(self._lse(0, self.off) - 1.0, 0.25, q_len)
        if self.off <= edge < kv_len:
            self.k[edge:edge + 1] = self._along(self._lse(0, kv_len) + 3.0, 0.0, 1)
        if kv_len > PF_KT:   # the first key of tile 1 raises the running max (a skipped rescale is visible)
            self.k[PF_KT:PF_KT + 1] = self._along(self._lse(0, PF_KT) + 2.0, 0.0, 1)
        if kv_len > 1:       # the last key carries about half the last row's mass (a dropped last tile is visible)
            self.k[kv_len - 1:] = self._along(self._lse(0, kv_len - 1), 0.0, 1)

    def _lse(self, lo, hi, rows=64):
        """Median log-sum-exp (natural log) of the scores of the first `rows` query tokens over keys [lo, hi) (unmasked)."""
        if hi <= lo:
            return 0.0
        q = self.q[:rows].double().reshape(-1, self.Hkv, self.G, d)
        z = torch.einsum("thgd,khd->thgk", q, self.k[lo:hi].double()) / RD
        return float(torch.logsumexp(z, -1).median())

    def _along(self, score, noise, count):
        """count keys (count, Hkv, d) along the group directions with about that score for the queries."""
        lam = score / (self.qscale * RD)
        return (noise * torch.randn((count, self.Hkv, d), generator=self.g, device=self.dev, dtype=torch.float64)
                + lam * RD * self.u[None]).bfloat16()

    def perturbations(self):
        names = ["limit_minus_1", "drop_last_tile"]
        if self.q_len > 1:             # (the last row sees every key already)
            names.append("limit_plus_1")
        if self.kv_len > PF_KT:        # (one tile: nothing to rescale)
            names.append("skip_rescale")
        if self.q_len < self.kv_len:
            names.append("top_left")
        if self.G > 1 and self.Hkv > 1:   # (with one kv-head both maps read head 0)
            names.append("head_mod")
        return names

    def restate(self, tokens=None, variant=None, block=1 << 25):
        """fp64 output (n, Hq, d) of the query tokens `tokens` (a LongTensor; None: all) under an optional perturbation:
          limit_plus_1 / limit_minus_1  every row sees one key more / fewer;
          top_left                      query i sees keys [0, i] (top-left alignment);
          head_mod                      q-head h reads kv-head h mod Hkv instead of h / G;
          drop_last_tile                the last key tile (the partial one when kv_len % 128 != 0) is left out;
          skip_rescale                  the online softmax over 128-key tiles leaves out one tile's rescale (the worst one)."""
        tok = torch.arange(self.q_len) if tokens is None else tokens
        tok = tok.to(self.dev)
        n, G = tok.numel(), self.G
        lim = tok + (0 if variant == "top_left" else self.off)
        lim = lim + {"limit_plus_1": 1, "limit_minus_1": -1}.get(variant, 0)
        keep_to = self.kv_len
        if variant == "drop_last_tile":
            keep_to = (self.kv_len - 1) // PF_KT * PF_KT
        ar = torch.arange(self.kv_len, device=self.dev)
        o = torch.empty((n, self.Hq, d), dtype=torch.float64, device=self.dev)
        rows = max(1, block // self.kv_len)
        for hq in range(self.Hq):
            hk = hq % self.Hkv if variant == "head_mod" else hq // G
            Kh, Vh = self.k[:, hk].double(), self.v[:, hk].double()
            for r0 in range(0, n, rows):
                qq = self.q[tok[r0:r0 + rows], hq].double()
                z = (qq @ Kh.t()) / RD
                vis = (ar[None] <= lim[r0:r0 + rows, None]) & (ar[None] < keep_to)
                z = z.masked_fill(~vis, -math.inf)
                if variant == "skip_rescale":
                    o[r0:r0 + rows, hq] = skip_rescale_rows(z, Vh)
                else:
                    p = torch.softmax(z, -1).nan_to_num(0.0)   # a row with no visible key: output 0
                    o[r0:r0 + rows, hq] = p @ Vh
        return o

    def check_inputs(self, tokens=None, probe=None):
        """Before any library call: every named perturbation moves some checked row by >= 10x the bar.  probe: the tokens the
        perturbations are evaluated on (default: the checked ones).  Returns the restatement of `tokens` and {name: movement}."""
        o = self.restate(tokens)
        assert bool(torch.isfinite(o).all())
        probe = tokens if probe is None else probe
        o_p = o if probe is tokens else self.restate(probe)
        moved = {}
        for name in self.perturbations():
            moved[name] = rel_rows(self.restate(probe, name), o_p)
            assert moved[name] >= 10 * BAR, f"{self.regime} ({self.q_len}, {self.kv_len}): '{name}' moves the output by {moved[name]:.2e} only"
        return o, moved


def skip_rescale_rows(z, V, tile=PF_KT):
    """Rows of scores z (R, n) over values V (n, d), fp64, as a tiled online softmax computes them when it leaves out the rescale
    of the running state at one tile: every key before that tile keeps a weight too large by e^jump, jump = how far the running
    max rises there.  The tile is the one where that matters most (largest excess weight), per row (fp64.softmax_state, batched)."""
    R, n = z.shape
    zp = F.pad(z, (0, (-n) % tile), value=-math.inf)
    m = z.max(1, keepdim=True).values
    e = torch.exp(zp - m).nan_to_num(0.0)
    run = torch.cummax(zp.reshape(R, -1, tile).max(2).values, 1).values
    if run.shape[1] > 1:
        jumps = (run[:, 1:] - run[:, :-1]).nan_to_num(0.0).clamp(max=700.0)
        before = torch.cumsum(e.reshape(R, -1, tile).sum(2), 1)[:, :-1]
        t = (torch.expm1(jumps) * before).argmax(1) + 1
        factor = torch.exp(jumps.gather(1, (t - 1)[:, None]))
        idx = torch.arange(zp.shape[1], device=z.device)
        e = torch.where(idx[None] < (t * tile)[:, None], e * factor, e)
    e = e[:, :n]
    return (e @ V) / e.sum(1, keepdim=True).clamp_min(1e-300)
