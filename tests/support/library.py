"""Helpers of the GPU tests that call the library: the two-layer context most tests run on, readers of its raw LSH tables and
probe lists, and the filled contexts several files share.  The native library is loaded inside the functions only, so
importing this module does not touch it or CUDA."""
import ctypes

import pytest
import torch

from magicpig_b200 import synth
from tests.support.fp64 import assert_1e3_f32, oracle_decode

DEV = "cuda:0"
d, NS, NL = 128, 4, 64


def two_layer_context(K, L, Hq, Hkv, B, M, gen, hf=None, options=None, **kw):
    """A Context of two layers on DEV, layer 0 dense and layer 1 sparse, head_dim d, NS sink and NL local rows, generation
    buffer gen.  kw: Context's keyword arguments; options: the set_option calls, in order; hf: the hash function to set."""
    from magicpig_b200.ops import Context
    ctx = Context(K, L, 2, Hq, Hkv, d, B, M, NS, NL, gen, dense_layers=[0], device=DEV, **kw)
    for key, val in (options or {}).items():
        ctx.set_option(key, val)
    if hf is not None:
        ctx.set_hash_func(hf.to(DEV))
    return ctx


def skip_unless_132_sms():
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the pinned paths are those of a 132-SM H100")


class _DevArray:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2}


def lsh_tables(ctx, layer):
    """Copies of the raw tables of `layer`: offsets int32 (C, Hkv, L, S, NB+1) and items (C, Hkv, L, M) as int64 in
    [0, 65536), C = ctx.num_contexts."""
    from magicpig_b200 import _native as N
    off, it = ctypes.c_void_p(), ctypes.c_void_p()
    N.check(ctx.lib.mpig_lsh_table_ptrs(ctx._h, layer, ctypes.byref(off), ctypes.byref(it)), "mpig_lsh_table_ptrs")
    S, C = ctx.get_info("table_segments"), ctx.num_contexts
    torch.cuda.synchronize()
    o = torch.as_tensor(_DevArray(off.value, (C, ctx.Hkv, ctx.L, S, ctx.NB + 1), "<i4"), device=DEV).clone()
    i = torch.as_tensor(_DevArray(it.value, (C, ctx.Hkv, ctx.L, ctx.M), "<i2"), device=DEV).clone()
    return o, (i.int() & 0xFFFF).long()


def assert_tables_equal(a, b, rows=None):
    """a, b: (offsets, items) as lsh_tables returns them, or slots of them; rows: the leading rows (slots) to compare, None:
    the whole arrays.  Identical offsets; per (table row, segment, bucket) the same items as a set (a merge and a build may
    order a bucket differently): every position of a segment's item range gets the key (bucket << 16 | item), and sorting
    these per table row must give the same sequence on both sides."""
    (oa, ia), (ob, ib) = a, b
    parts = [("", oa, ia, ob, ib)] if rows is None else [(f"slot {r}: ", oa[r], ia[r], ob[r], ib[r]) for r in rows]
    for what, oa, ia, ob, ib in parts:
        assert torch.equal(oa, ob), f"{what}offsets differ"
        o = oa.reshape(-1, oa.shape[-2], oa.shape[-1]).long()          # (table rows, S, NB+1)
        xa, xb = ia.reshape(o.shape[0], -1).long(), ib.reshape(o.shape[0], -1).long()
        S, NB = o.shape[1], o.shape[2] - 1
        p = torch.arange(xa.shape[1], device=o.device)[None].expand(o.shape[0], -1).contiguous()
        for s in range(S):
            bucket = torch.searchsorted(o[:, s, :NB].contiguous(), p, right=True) - 1
            valid = (p >= o[:, s, :1]) & (p < o[:, s, NB:])
            ka = torch.where(valid, (bucket << 16) | xa, -1).sort(dim=1).values
            kb = torch.where(valid, (bucket << 16) | xb, -1).sort(dim=1).values
            assert torch.equal(ka, kb), f"{what}segment {s}: bucket contents differ"


def assert_lists_equal(nnz_a, res_a, nnz_b, res_b):
    """Equal nnz and, per row, equal index lists (the first nnz entries)."""
    assert torch.equal(nnz_a, nnz_b), "nnz differ"
    valid = torch.arange(res_a.shape[1], device=DEV)[None] < nnz_a[:, None]
    assert torch.equal(torch.where(valid, res_a, -1), torch.where(valid, res_b, -1)), "index lists differ"


class _Cfg:
    """A small Llama-shaped config for the drop-in class."""
    num_hidden_layers = 3
    num_key_value_heads = 2
    num_attention_heads = 8
    hidden_size = 8 * 128


class Doc:
    """One context: offloaded keys of one request, its window and its dense-layer prefix (CPU tensors)."""

    def __init__(self, Hkv, n, K, L, hf, seed, w=NS + NL, P_dense=300, on_gpu=False):
        self.n, self.w = n, w
        if on_gpu:
            g = torch.Generator(device=DEV).manual_seed(seed)
            self.key = torch.randn((Hkv, n, d), generator=g, device=DEV).bfloat16()
            self.value = torch.randn((Hkv, n, d), generator=g, device=DEV).bfloat16()
            self.kn = self.key.float().norm(p=2, dim=-1)
            self.avg = torch.zeros((Hkv, d), dtype=torch.bfloat16)
            self.kcodes = None
        else:
            key, value, kn, avg = synth.make_kv(1, Hkv, n, d, seed=seed, dist="gauss")
            self.key, self.value, self.kn, self.avg = key[0], value[0], kn[0], avg[0].reshape(Hkv, d)
            self.kcodes = synth.hash_keys(key, hf, K, L)[0]
        g = torch.Generator().manual_seed(seed + 1)
        self.wk = torch.randn((Hkv, w, d), generator=g).bfloat16()
        self.wv = torch.randn((Hkv, w, d), generator=g).bfloat16()
        self.dk = torch.randn((P_dense, Hkv, d), generator=g).bfloat16()
        self.dv = torch.randn((P_dense, Hkv, d), generator=g).bfloat16()

    def fill_store(self, ctx, b):
        kd = self.key.to(DEV).contiguous()
        ctx.attn_fill(1, b, kd, self.value.to(DEV).contiguous(), self.kn.to(DEV).contiguous())
        ctx.lsh_build(1, b, ctx.hash_keys(kd) if self.kcodes is None else self.kcodes.to(DEV).contiguous())

    def fill_request(self, ctx, b):
        ctx.window_fill(1, b, self.avg.to(DEV).contiguous(), self.wk.to(DEV).contiguous(), self.wv.to(DEV).contiguous())
        ctx.dense_fill(0, b, self.dk.to(DEV), self.dv.to(DEV), self.dk.shape[0])


class Run:
    """One context with a sparse layer 1 (layer 0 dense) filled from seeded keys, and the window history on the host."""

    def __init__(self, B, Hq, Hkv, n, K, L, M, gen, seed, route="build", on_gpu=False, w0=NS + NL, impl=1):
        self.B, self.Hq, self.Hkv, self.n, self.K, self.L, self.M, self.G = B, Hq, Hkv, n, K, L, M, Hq // Hkv
        self.hf = synth.make_hash_func(d, K, L, seed=seed)
        self.g = torch.Generator().manual_seed(seed + 1)
        if on_gpu:   # full-size keys are drawn on the device
            gg = torch.Generator(device=DEV).manual_seed(seed + 2)
            self.key = torch.randn((B, Hkv, n, d), generator=gg, device=DEV).bfloat16()
            self.value = torch.randn((B, Hkv, n, d), generator=gg, device=DEV).bfloat16()
            self.kn = self.key.norm(p=2, dim=-1).float()
            self.avg = torch.zeros((B, Hkv, 1, d), dtype=torch.bfloat16)
        else:
            self.key, self.value, self.kn, self.avg = synth.make_kv(B, Hkv, n, d, seed=seed + 2, dist="gauss")
        self.wk = torch.randn((B, Hkv, w0, d), generator=self.g).bfloat16()
        self.wv = torch.randn((B, Hkv, w0, d), generator=self.g).bfloat16()
        self.ctx = two_layer_context(K, L, Hq, Hkv, B, M, gen, self.hf, dict(decode_impl=impl, out_f32=1))
        for b in range(B):
            kb = self.key[b].to(DEV).contiguous()
            self.ctx.attn_fill(1, b, kb, self.value[b].to(DEV).contiguous(), self.kn[b].to(DEV).contiguous())
            codes = self.ctx.hash_keys(kb)
            if route == "sorted":
                sc, si = codes.sort()
                self.ctx.lsh_fill(1, b, sc.contiguous(), si.int().contiguous())
            else:
                self.ctx.lsh_build(1, b, codes)
            self.ctx.window_fill(1, b, self.avg[b].reshape(Hkv, d).to(DEV), self.wk[b].to(DEV), self.wv[b].to(DEV))
        self.n_off = n   # offloaded keys per request

    def token(self, q=None):
        """One eager decode step (plan + layer-1 decode); the window history gains the centred key."""
        B, Hq, Hkv = self.B, self.Hq, self.Hkv
        if q is None:
            q = torch.randn((B, Hq, 1, d), generator=self.g).bfloat16()
        k_new = torch.randn((B, Hkv, 1, d), generator=self.g).bfloat16()
        v_new = torch.randn((B, Hkv, 1, d), generator=self.g).bfloat16()
        self.ctx.plan()
        out = self.ctx.decode(1, q.to(DEV), k_new.to(DEV), v_new.to(DEV))
        return q, k_new, v_new, out

    def push(self, k_new, v_new):
        self.wk = torch.cat([self.wk, k_new - self.avg], dim=2)
        self.wv = torch.cat([self.wv, v_new], dim=2)

    def spill(self, keep=NL):
        """Spill through the context and apply the same semantics to the host history; returns the spilled rows."""
        got = self.ctx.spill_window(keep)
        w = self.wk.shape[2]
        g = max(0, w - NS - keep)
        assert got.tolist() == [g] * self.B
        rows = (self.wk[:, :, NS:NS + g], self.wv[:, :, NS:NS + g])
        if g:
            self.wk = torch.cat([self.wk[:, :, :NS], self.wk[:, :, NS + g:]], dim=2)
            self.wv = torch.cat([self.wv[:, :, :NS], self.wv[:, :, NS + g:]], dim=2)
        self.n_off += g
        return g, rows

    def rebuild(self):
        """A second context whose layer-1 tables are built by mpig_lsh_build over the keys the first one now stores."""
        k_st, _, _ = self.ctx.read_cache(1, True, False, False)
        other = two_layer_context(self.K, self.L, self.Hq, self.Hkv, self.B, self.M, 8, self.hf)
        for b in range(self.B):
            other.lsh_build(1, b, self.ctx.hash_keys(k_st[b, :, : self.n_off].contiguous()))
        return other

    def check_decode(self, q, k_new, v_new, out_f32):
        """Oracle on exactly the stored state (keys, norms, codes of the stored keys), n = all offloaded keys."""
        n = self.n_off
        k_st, v_st, kn_st = (x.cpu() for x in self.ctx.read_cache(1))
        k_dev = k_st[:, :, :n].contiguous()
        kcodes = torch.stack([self.ctx.hash_keys(k_dev[b].to(DEV)).cpu() for b in range(self.B)])
        t = dict(B=self.B, Hq=self.Hq, Hkv=self.Hkv, d=d, K=self.K, L=self.L, n=n, M=self.M, hash_func=self.hf, kcodes=kcodes,
                 key=k_dev, value=v_st[:, :, :n].contiguous(), key_norm=kn_st[:, :, :n].contiguous(), avg_k=self.avg)
        _, nz_ref, _, o_exact = oracle_decode(t, q, k_new, v_new, self.wk, self.wv, self.G)
        nnz, _ = self.ctx.last_probe()
        assert torch.equal(nnz.cpu(), nz_ref)
        assert_1e3_f32(out_f32, o_exact)


class Twins:
    """Two identically filled contexts (sparse layer 1, dense layer 0): `tok` runs T-token steps, `seq` single-token steps.
    Request b's window starts with NS + NL - 5*b rows."""

    def __init__(self, B, Hq, Hkv, n, K, L, T, seed, gen=32, P_dense=300, on_gpu=False):
        self.B, self.Hq, self.Hkv, self.n, self.K, self.L, self.G = B, Hq, Hkv, n, K, L, Hq // Hkv
        self.M = max(n, P_dense) + 256
        self.hf = synth.make_hash_func(d, K, L, seed=seed)
        self.g = torch.Generator().manual_seed(seed + 1)
        if on_gpu:
            gg = torch.Generator(device=DEV).manual_seed(seed + 2)
            self.key = torch.randn((B, Hkv, n, d), generator=gg, device=DEV).bfloat16()
            self.value = torch.randn((B, Hkv, n, d), generator=gg, device=DEV).bfloat16()
            self.kn = self.key.norm(p=2, dim=-1).float()
            self.avg = torch.zeros((B, Hkv, 1, d), dtype=torch.bfloat16)
            self.kcodes = None
        else:
            qd = synth.make_query(B, Hq, d, seed=seed + 3).reshape(B, Hkv, self.G, d)[:, :, 0].float()
            # K10 L150 samples few keys of i.i.d. Gaussian data: keys clustered around query directions, as test_fused_decode
            dist = "clustered" if K >= 10 else "gauss"
            self.key, self.value, self.kn, self.avg = synth.make_kv(B, Hkv, n, d, seed=seed + 2, dist=dist, q_dirs=qd)
            self.kcodes = synth.hash_keys(self.key, self.hf, K, L)
        self.win = [(torch.randn((Hkv, NS + NL - 5 * b, d), generator=self.g).bfloat16(),
                     torch.randn((Hkv, NS + NL - 5 * b, d), generator=self.g).bfloat16()) for b in range(B)]
        self.dk = torch.randn((B, P_dense, Hkv, d), generator=self.g).bfloat16()
        self.dv = torch.randn((B, P_dense, Hkv, d), generator=self.g).bfloat16()
        self.ctxs = []
        for tmax in (T, 1):
            ctx = two_layer_context(K, L, Hq, Hkv, B, self.M, gen, self.hf, dict(save_mask=1, out_f32=1), alloc_dense_kv=True,
                                    max_query_tokens=tmax)
            for b in range(B):
                kb = self.key[b].to(DEV).contiguous()
                ctx.attn_fill(1, b, kb, self.value[b].to(DEV).contiguous(), self.kn[b].to(DEV).contiguous())
                ctx.lsh_build(1, b, self.kcodes[b].to(DEV) if self.kcodes is not None else ctx.hash_keys(kb))
                ctx.window_fill(1, b, self.avg[b].reshape(Hkv, d).to(DEV), self.win[b][0].to(DEV), self.win[b][1].to(DEV))
                ctx.dense_fill(0, b, self.dk[b].to(DEV), self.dv[b].to(DEV), P_dense)
            self.ctxs.append(ctx)
        self.tok, self.seq = self.ctxs

    def inputs(self, T):
        B, Hq, Hkv = self.B, self.Hq, self.Hkv
        q = torch.randn((B, T, Hq, d), generator=self.g).bfloat16()
        k = torch.randn((B, T, Hkv, d), generator=self.g).bfloat16()
        v = torch.randn((B, T, Hkv, d), generator=self.g).bfloat16()
        return q, k, v
