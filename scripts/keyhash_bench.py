"""Throughput of the wgmma key-hash kernel at the BASELINE shape (8 KV heads x 98K keys, K=10, L=150) against the
torch bf16 GEMM + sign-pack glue the reference uses (attnserver.py:159-168).   python scripts/keyhash_bench.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicpig_b200 import synth  # noqa: E402
from magicpig_b200.ops import Context  # noqa: E402

dev = "cuda:0"
K, L, Hkv, d, n = 10, 150, 8, 128, 97932
ctx = Context(K, L, 1, 32, Hkv, d, 1, 98304, device=dev)
hf = synth.make_hash_func(d, K, L, seed=1).to(dev)
ctx.set_hash_func(hf)
keys = torch.randn((Hkv, n, d), device=dev).bfloat16()
out = torch.empty((Hkv, L, n), dtype=torch.int16, device=dev)


def timeit(fn, reps=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


flop = 2.0 * Hkv * n * d * K * L
for impl in (1, 0):
    ctx.set_option("keyhash_impl", impl)
    ms = timeit(lambda: ctx.hash_keys(keys, out=out))
    print(f"mpig_hash_keys impl={impl} (wgmma): {ms * 1e3:8.1f} us   {flop / ms / 1e9:7.1f} TFLOP/s   out {out.numel() * 2 / 1e6:.0f} MB -> {out.numel() * 2 / ms / 1e6:.0f} GB/s")
ctx.set_option("keyhash_impl", 1)
for sk in (1, 2, 3, 4, 7):
    ctx.set_option("keyhash_skip", sk)
    ms = timeit(lambda: ctx.hash_keys(keys, out=out))
    print(f"  skip={sk} (1 no stores, 2 no sign pack, 4 no MMAs): {ms * 1e3:8.1f} us")
ctx.set_option("keyhash_skip", 0)
out.zero_()
ctx.hash_keys(keys, out=out)
ms2 = timeit(lambda: synth.hash_keys(keys, hf, K, L), reps=3)
print(f"torch GEMM + pack glue  : {ms2 * 1e3:8.1f} us   {flop / ms2 / 1e9:7.1f} TFLOP/s")
ref = synth.hash_keys(keys, hf, K, L)
print("mismatching codes vs torch bf16-GEMM path:", int((ref != out).sum()), "of", out.numel())

# the rest of the device-side table build (SURVEY 8(f)-1): counting sort into the bucketed tables, and the
# reference-style route (torch sort + mpig_lsh_fill) for comparison
ms = timeit(lambda: ctx.lsh_build(0, 0, out), reps=5)
print(f"mpig_lsh_build (counting sort, {Hkv}x{L} tables of {n} keys): {ms * 1e3:8.1f} us   "
      f"({(out.numel() * 2 + out.numel() * 4) / ms / 1e6:.0f} GB/s of codes-in + items-out)")


def sorted_route():
    sc, si = out.sort()
    ctx.lsh_fill(0, 0, sc, si.int())


ms = timeit(sorted_route, reps=2)
print(f"torch sort + mpig_lsh_fill (attnserver.py:186-193 route): {ms * 1e3:8.1f} us")
