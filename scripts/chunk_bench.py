"""Chunk steps on the H100: per-layer chunk-attention time (sparse and dense layers) and the end-to-end prompt rate of
LlamaDecodeRunner.extend() against feeding the same turn through the captured single-token step.

Shape: Llama-3.1-8B (Hq/Hkv = 32/8, d = 128), P = 98 000 prompt tokens, K = 10, L = 150.  Kernel lines at B = 1 and at B = 8 requests
forked from one shared context (shared spill).  Writes profiles/h100_chunk_line.json (or --out) with the card's name and power limit
read in the same run.

  python scripts/chunk_bench.py [--out profiles/h100_chunk_line.json] [--P 98000] [--layers 32]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from magicpig_b200 import synth  # noqa: E402
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner  # noqa: E402
from magicpig_b200.ops import Context  # noqa: E402

DEV = "cuda:0"
PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35   # H100 SXM data sheet: dense BF16, HBM3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def kernel_lines(B, P, shared, Ts, reps=20):
    Hq, Hkv, d, K, L = 32, 8, 128, 10, 150
    M = P + 2048
    ctx = Context(K, L, 2, Hq, Hkv, d, B, M, 4, 64, 1100, dense_layers=[0], alloc_dense_kv=True, device=DEV,
                  num_contexts=1 if shared else 0, shared_spill=shared)
    ctx.set_hash_func(synth.make_hash_func(d, K, L, seed=1).to(DEV))
    ctx.reserve_chunk_tokens(max(Ts))
    g = torch.Generator(device=DEV).manual_seed(2)
    n = P - 68
    for r in (range(1) if shared else range(B)):
        k = torch.randn((Hkv, n, d), generator=g, device=DEV).bfloat16()
        v = torch.randn((Hkv, n, d), generator=g, device=DEV).bfloat16()
        ctx.attn_fill(1, r, k, v, k.float().norm(dim=-1).contiguous())
        ctx.lsh_build(1, r, ctx.hash_keys(k))
        kd = torch.randn((P, Hkv, d), generator=g, device=DEV).bfloat16()
        ctx.dense_fill(0, r, kd, kd, P)
        w = torch.randn((Hkv, 68, d), generator=g, device=DEV).bfloat16()
        ctx.window_fill(1, r, torch.zeros((Hkv, d), dtype=torch.bfloat16, device=DEV), w, w)
        del k, v, kd
    if shared:
        for b in range(1, B):
            ctx.fork(0, b)
    lines = []
    for T in Ts:
        q = torch.randn((B, T, Hq, d), generator=g, device=DEV).bfloat16()
        kv = torch.randn((B, T, Hkv, d), generator=g, device=DEV).bfloat16()
        ctx.plan_chunk(T)
        for layer, kind in ((1, "sparse"), (0, "dense")):
            out = ctx.chunk_attend(layer, T, q, kv, kv)   # warm-up (module load, attributes)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):   # the same step again: the rows land where they did
                ctx.chunk_attend(layer, T, q, kv, kv, out)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            ctx_keys = (n + 68) if kind == "sparse" else P   # keys before the chunk per request
            G = Hq // Hkv
            # 4*d FLOP per (query row, visible key): every row sees the context, token t also t + 1 chunk rows
            flop = 4 * d * B * Hkv * G * (T * ctx_keys + T * (T + 1) / 2)
            # algorithmic bytes: every record a request sees, once per kv-head (the m-blocks share them through L2), + q and out.
            # The sparse store is the slot's, read once for all requests of one shared context; the windows and (no dense tail here)
            # the dense caches are per request.
            if kind == "sparse":
                recs = Hkv * (n * (1 if shared else B) + B * (68 + T))
            else:
                recs = B * Hkv * (P + T)
            byts = recs * 512 + 2 * B * T * Hq * d * 2
            tf, tbs = flop / ms / 1e9, byts / ms / 1e9
            f_share, b_share = tf / PEAK_TFLOPS, tbs / PEAK_TBS
            lines.append(dict(B=B, shared=shared, T=T, layer=kind, ms=round(ms, 4), tflops=round(tf, 1), tb_per_s=round(tbs, 3),
                              flop_share=round(f_share, 3), byte_share=round(b_share, 3), share_of_peak=round(max(f_share, b_share), 3),
                              bound="compute" if f_share >= b_share else "memory"))
            print(json.dumps(lines[-1]), flush=True)
        ctx.rewind(torch.full((B,), T, dtype=torch.int32, device=DEV))
    ctx.close()
    torch.cuda.empty_cache()
    return lines


def extend_line(P, T_turn, layers):
    run = LlamaDecodeRunner(LLAMA31_8B, 10, 150, 1, P + 2 * T_turn + 512, device=DEV, seed=0, generation_buffer=1024,
                            num_layers=layers, max_chunk_tokens=1024)
    run.synthetic_prefill(P)
    ids = torch.randint(0, LLAMA31_8B.vocab_size, (1, T_turn), device=DEV)
    run.extend(ids[:, :8])   # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run.extend(ids)
    torch.cuda.synchronize()
    t_ext = time.perf_counter() - t0
    # the same turn through the captured single-token step (spilling when the window fills)
    run.server.spill_window()
    run.capture(warm=2)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    room = run.generation_buffer - 4
    for i in range(T_turn):
        if i % room == 0:
            torch.cuda.synchronize()
            run.server.spill_window()
        run.ids.copy_(ids[:, i:i + 1])
        run.replay()
    torch.cuda.synchronize()
    t_step = time.perf_counter() - t0
    return dict(P=P, turn_tokens=T_turn, layers=layers, extend_s=round(t_ext, 4), extend_tok_per_s=round(T_turn / t_ext, 1),
                step_s=round(t_step, 4), step_tok_per_s=round(T_turn / t_step, 1), speedup=round(t_step / t_ext, 2),
                error_flags=run.server.ctx.error_flags())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_chunk_line.json")
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--turn", type=int, default=1024)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("chunk_bench needs a GPU")
    res = dict(card=card(), card_fields="name, power.limit, clocks.max.sm", shape="Llama-3.1-8B K10 L150", kernels=[])
    res["kernels"] += kernel_lines(1, a.P, False, (64, 256, 1024))
    res["kernels"] += kernel_lines(8, a.P, True, (64, 256, 1024))
    res["extend"] = extend_line(a.P, a.turn, a.layers)
    print(json.dumps(res["extend"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(dict(card=res["card"])))


if __name__ == "__main__":
    main()
