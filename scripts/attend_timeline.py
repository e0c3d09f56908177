"""Stage timestamps (globaltimer, ns) of attend_mma_kernel warps: where does a warp's life go?"""
import ctypes, os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicpig_b200 import synth
from magicpig_b200.ops import Context

dev = "cuda:0"
B, Hq, Hkv, d, K, L, P = 1, 32, 8, 128, 10, 150, 98000
n, M, nl = P - 68, 98304, 3
ctx = Context(K, L, nl, Hq, Hkv, d, B, M, device=dev)
g = torch.Generator(device=dev).manual_seed(0)
hf = torch.randn((d, K * L), generator=g, device=dev).bfloat16()
ctx.set_hash_func(hf)
for l in range(nl):
    key = torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16()
    key = key - key.mean(dim=1, keepdim=True)
    ctx.attn_fill(l, 0, key, torch.randn((Hkv, n, d), generator=g, device=dev).bfloat16(), key.norm(p=2, dim=-1).float())
    ctx.lsh_build(l, 0, synth.hash_keys(key, hf, K, L))
H = B * Hq
q = torch.randn((nl, H, d), generator=g, device=dev).bfloat16()
res = [torch.zeros((H, M), dtype=torch.int32, device=dev) for _ in range(nl)]
nnz = [torch.zeros((H,), dtype=torch.int32, device=dev) for _ in range(nl)]
qn = []
for l in range(nl):
    c, qq = ctx.simhash(q[l]); qn.append(qq)
    ctx.lsh_batch_retrieve(l, c, res[l], nnz[l])
out = torch.zeros((H, d), dtype=torch.bfloat16, device=dev); mve = torch.zeros((2, H), device=dev)
ctx.set_option("attend_debug", 1)
import itertools
for frac, tma in itertools.product((1.0,), (1, 0)):
    ctx.set_option("attend_tma", tma)
    nz = [(x.float() * frac).int() for x in nnz]
    for l in range(nl):
        ctx.attention_wrapper(l, K, L, out, mve, q[l], qn[l], res[l], nz[l])
    torch.cuda.synchronize()
    for _ in range(300):  # sustained load so that the SM clock is at its working frequency
        for l in range(nl):
            ctx.attention_wrapper(l, K, L, out, mve, q[l], qn[l], res[l], nz[l])
    # run ONE more launch on a layer whose data is cold in L2
    nw = torch.cuda.get_device_properties(0).multi_processor_count * 12   # 12 warps per SM
    ctx.attention_wrapper(1, K, L, out, mve, q[1], qn[1], res[1], nz[1])
    ctx.attention_wrapper(2, K, L, out, mve, q[2], qn[2], res[2], nz[2])
    torch.cuda.synchronize()
    buf = np.zeros((nw, 16), dtype=np.uint64)
    rc = ctx.lib.mpig_debug_read(ctx._h, buf.ctypes.data_as(ctypes.c_void_p), nw)
    assert rc == 0
    t = buf.astype(np.int64)
    act = t[:, 3] > 0  # warps that processed a tile
    t0 = t[act, 0:1]  # per-warp start (clock64 is per SM)
    names = ["start", "prefix+sync", "copies issued", "tile landed", "QK done", "transform done", "softmax done", "PV done",
             "flush start", "level1 done", "published", "merged+written", "head resolved", "barrier armed", "bounds known", "idx addr ready"]
    print(f"--- frac={frac} tma={tma}: active warps {act.sum()} of {nw}; kernel span (max stamp - min start) = "
          f"n/a (per-warp cycle stamps)")
    for k in [0, 1, 12, 14, 13, 15, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11]:
        nm = names[k]
        col = t[act, k]
        v = (((col - t0[:, 0]) & 0xffffffff)[col > 0]) / 1.9  # 32-bit cycle stamps -> ns at 1.9 GHz
        if len(v):
            print(f"  [{k:2d}] {nm:16s} n={len(v):5d}  mean {v.mean() / 1e3:7.2f} us   p10 {np.percentile(v, 10) / 1e3:7.2f}   p90 {np.percentile(v, 90) / 1e3:7.2f}   max {v.max() / 1e3:7.2f}")
