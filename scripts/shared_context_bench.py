"""Batched decode over ONE shared context (context slots, mpig_config.num_contexts) -> one JSON line.

Llama-3.1-8B with random weights, a synthetic P-token context filled once (request 0) and forked to the other requests, K10
L150, one context slot (num_contexts = 1), B in {1, 2, 4, 8}, distinct token ids per request.  For every B: the captured step()
time (CUDA events, median over blocks of replays), aggregate tokens/s, the context's HBM bytes (mpig_device_bytes) and the
fused kernel's cluster waves.  Then B = 2 on one slot against B = 2 on two slots filled with the same context, alternated block by
block: logits must be bitwise equal; both step times are recorded.  The card's name and power limit are read in the same run.

    python scripts/shared_context_bench.py --out profiles/h100_shared_line.json
"""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def make(B, C, P, M, K, L, gen):
    r = LlamaDecodeRunner(LLAMA31_8B, K, L, B, M, device=DEV, seed=0, generation_buffer=gen, num_contexts=C)
    r.synthetic_prefill(P, shared=True)
    r.ids.copy_(torch.arange(1, B + 1, device=DEV)[:, None] * 1009)   # distinct ids per request
    r.capture()
    return r


def time_block(r, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        r.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def median(x):
    x = sorted(x)
    return x[len(x) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--M", type=int, default=98304)
    ap.add_argument("--K", type=int, default=10)
    ap.add_argument("--L", type=int, default=150)
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--blocks", type=int, default=7)
    ap.add_argument("--per-block", type=int, default=20)
    ap.add_argument("--pair-P", type=int, default=49000, help="context of the one-slot / two-slot pair (two stores must fit beside two models)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device (an H100); nothing is measured without one")
    gen = 16 + args.blocks * args.per_block * 2 + 8   # window rows the warm-up, capture and replays use
    line = {"workload": f"Llama-3.1-8B random weights, synthetic shared context P={args.P}, K{args.K} L{args.L}, num_contexts=1",
            "card": card(), "runs": []}
    for B in [int(x) for x in args.batches.split(",")]:
        r = make(B, 1, args.P, args.M, args.K, args.L, gen)
        ctx = r.server.ctx
        for _ in range(10):
            r.replay()
        ms = median([time_block(r, args.per_block) for _ in range(args.blocks)])
        line["runs"].append({"B": B, "num_contexts": ctx.num_contexts, "step_ms": round(ms, 4), "tokens_per_s": round(B * 1000.0 / ms, 1),
                             "device_bytes": ctx.device_bytes, "fused_cluster_waves": ctx.get_info("fused_cluster_waves"),
                             "max_memory_allocated": torch.cuda.max_memory_allocated()})
        print(json.dumps(line["runs"][-1]), flush=True)
        del r, ctx
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    # B = 2: one slot against two slots holding the same context, alternated
    Mp = ((args.pair_P + 64 + 1023) // 1024) * 1024
    runners = {C: make(2, C, args.pair_P, Mp, args.K, args.L, gen) for C in (1, 2)}
    times = {1: [], 2: []}
    for _ in range(10):
        for C in (1, 2):
            runners[C].replay()
    equal = torch.equal(runners[1].logits, runners[2].logits)
    for _ in range(args.blocks):
        for C in (1, 2):
            times[C].append(time_block(runners[C], args.per_block))
        equal &= torch.equal(runners[1].logits, runners[2].logits)
    line["pair"] = {"B": 2, "P": args.pair_P, "M": Mp, "logits_bitwise_equal": bool(equal),
                    "step_ms": {f"num_contexts={C}": round(median(times[C]), 4) for C in (1, 2)},
                    "block_ms": {f"num_contexts={C}": [round(t, 4) for t in times[C]] for C in (1, 2)},
                    "device_bytes": {f"num_contexts={C}": runners[C].server.ctx.device_bytes for C in (1, 2)}}
    print(json.dumps(line["pair"]), flush=True)
    line["card_after"] = card()
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")
    if not equal:
        raise SystemExit("one-slot and two-slot logits differ")


if __name__ == "__main__":
    main()
