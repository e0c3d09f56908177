"""Per-kernel timing of the three hot-path kernels at the BASELINE shape, outside the model.

Several layers of distinct synthetic data (so every launch misses L2), launches enqueued back to back,
CUDA events around each batch.  Used to compare kernel variants / tuning knobs on the GPU box:

    python scripts/kernel_bench.py [--B 1] [--P 98000] [--layers 6] [--reps 20]
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicpig_b200 import synth  # noqa: E402
from magicpig_b200.ops import Context  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--B", type=int, default=1)
ap.add_argument("--P", type=int, default=98000)
ap.add_argument("--K", type=int, default=10)
ap.add_argument("--L", type=int, default=150)
ap.add_argument("--layers", type=int, default=6)
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--fracs", default="")
ap.add_argument("--variants", default="tma=1,warps=12;tma=0,warps=12;tma=1,warps=8;tma=0,warps=8;tma=1,warps=6;tma=0,warps=6")
args = ap.parse_args()

dev = "cuda:0"
B, Hq, Hkv, d, K, L = args.B, 32, 8, 128, args.K, args.L
n = args.P - 68
M = ((args.P + 255) // 256) * 256 + 256
H = B * Hq
nl = args.layers
ctx = Context(K, L, nl, Hq, Hkv, d, B, M, device=dev)
g = torch.Generator(device=dev).manual_seed(0)
hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
ctx.set_hash_func(hf)
t0 = time.time()
for l in range(nl):
    for b in range(B):
        key = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
        key = key - key.mean(dim=1, keepdim=True)
        val = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
        kn = key.norm(p=2, dim=-1).float()
        ctx.attn_fill(l, b, key, val, kn)
        ctx.lsh_build(l, b, synth.hash_keys(key, hf, K, L))
        ctx.window_fill(l, b, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=dev),
                        torch.randn((Hkv, 68, d), generator=g, device=dev).bfloat16(),
                        torch.randn((Hkv, 68, d), generator=g, device=dev).bfloat16())
torch.cuda.synchronize()
print(f"setup {time.time() - t0:.1f}s, context {ctx.device_bytes / 1e9:.1f} GB")
q = torch.randn((nl, H, d), generator=g, device=dev).bfloat16()
codes = [None] * nl
qn = [None] * nl
res = [torch.zeros((H, M), dtype=torch.int32, device=dev) for _ in range(nl)]
nnz = [torch.zeros((H,), dtype=torch.int32, device=dev) for _ in range(nl)]
for l in range(nl):
    codes[l], qn[l] = ctx.simhash(q[l])
    ctx.lsh_batch_retrieve(l, codes[l], res[l], nnz[l])
torch.cuda.synchronize()
tot = sum(int(x.sum()) for x in nnz) / nl
print(f"mean nnz/head {tot / H:.0f} ({tot / H / n * 100:.2f}% of n)")
out = torch.zeros((H, d), dtype=torch.bfloat16, device=dev)
mve = torch.zeros((2, H), dtype=torch.float32, device=dev)


def timeit(fn, reps):
    """fn(l) enqueues one launch on layer l.  nl*reps launches are captured into ONE CUDA graph (no Python / launch
    overhead between kernels) and the graph is replayed; returns mean us per launch."""
    for l in range(nl):
        fn(l)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for l in range(nl):
            fn(l)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        for _ in range(reps):
            for l in range(nl):
                fn(l)
    gr.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        gr.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (3 * reps * nl)


codes_out = torch.zeros((H, L), dtype=torch.int32, device=dev)
qn_out = torch.zeros((H,), dtype=torch.float32, device=dev)
import ctypes
from magicpig_b200 import _native as N_


def simhash_raw(l):
    N_.check(ctx.lib.mpig_simhash(ctx._h, ctypes.c_void_p(q[l].data_ptr()), ctypes.c_void_p(codes_out.data_ptr()),
                                  ctypes.c_void_p(qn_out.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))


us = timeit(simhash_raw, args.reps)
print(f"simhash  {us:7.2f} us/launch")
us = timeit(lambda l: ctx.lsh_batch_retrieve(l, codes[l], res[l], nnz[l]), args.reps)
pb = H * L * (8 + 4 * n / (1 << K)) + 4 * tot
print(f"probe    {us:7.2f} us/launch   {pb / us / 1e3:7.1f} GB/s algorithmic")
ab = tot * 520 + H * 520
for var in args.variants.split(";"):
    kv = dict(x.split("=") for x in var.split(","))
    ctx.set_option("attend_tma", int(kv.get("tma", 1)))
    ctx.set_option("attend_warps", int(kv.get("warps", 12)))
    ctx.set_option("attend_ctas", int(kv.get("ctas", 0)))
    try:
        us = timeit(lambda l: ctx.attention_wrapper(l, K, L, out, mve, q[l], qn[l], res[l], nnz[l]), args.reps)
        print(f"attend [{var:28s}] {us:7.2f} us/launch   {ab / us / 1e3:7.1f} GB/s algorithmic ({ab / 1e6:.1f} MB)")
    except Exception as e:
        print(f"attend [{var}] failed: {e}")

# how does attend scale with the amount of work?  (separates fixed latency from throughput)
if args.fracs:
    ctx.set_option("attend_tma", 1); ctx.set_option("attend_warps", 12)
    for f in [float(x) for x in args.fracs.split(",")]:
        nnz_f = [(x.float() * f).int() for x in nnz]
        tot_f = sum(int(x.sum()) for x in nnz_f) / nl
        us = timeit(lambda l: ctx.attention_wrapper(l, K, L, out, mve, q[l], qn[l], res[l], nnz_f[l]), args.reps)
        print(f"attend frac={f:4.2f} rows={tot_f:8.0f} {us:7.2f} us/launch  {(tot_f * 520) / us / 1e3:7.1f} GB/s")

# attribute the attend time by elimination (results are wrong in these modes: timing only)
if args.fracs:
    for sk, nm in [(0, "full"), (4, "no merges"), (2, "no tile math"), (6, "no math, no merges"), (1, "no row fetch"), (3, "no fetch, no math"), (7, "prologue + index loads only"), (8, "no QK mma"), (16, "no LSH transform"), (32, "no PV mma"), (56, "no QK, transform, PV")]:
        ctx.set_option("attend_skip", sk)
        us = timeit(lambda l: ctx.attention_wrapper(l, K, L, out, mve, q[l], qn[l], res[l], nnz[l]), args.reps)
        print(f"attend skip={sk} ({nm:28s}) {us:7.2f} us/launch")
    ctx.set_option("attend_skip", 0)

# fused per-layer decode (simhash+append -> probe -> attend with PDL), graph-captured
kn_ = torch.randn((nl, B * Hkv, d), generator=g, device=dev).bfloat16()
vn_ = torch.randn((nl, B * Hkv, d), generator=g, device=dev).bfloat16()
out2 = torch.zeros((B, Hq * d), dtype=torch.bfloat16, device=dev)
ctx.plan()
for var in ["tma=1,warps=12", "tma=0,warps=12"]:
    kv = dict(x.split("=") for x in var.split(","))
    ctx.set_option("attend_tma", int(kv.get("tma", 1)))
    ctx.set_option("attend_warps", int(kv.get("warps", 12)))
    us = timeit(lambda l: ctx.decode(l, q[l], kn_[l], vn_[l], out2), args.reps)
    print(f"decode [{var:28s}] {us:7.2f} us/layer  (3 kernels, PDL)")
