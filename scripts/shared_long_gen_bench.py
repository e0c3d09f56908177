"""Long generation of a batch that shares one context: the captured Llama-3.1-8B decode step (synthetic weights, K = 10, L = 150)
for B requests forked from one P-token prompt in one context slot, with dense_tail_rows R, replayed for N generated tokens per
request in two arms:

  a  shared spill (mpig_config.shared_spill), generation_buffer = 256 (--gen-buf): spill_window() between replays whenever the
     window is full; each request's spilled tokens go into the shared store and tables, private to it
  b  generation_buffer = N + 8, no spill: every sparse layer attends the whole generation densely

Per arm: ms per step over the whole generation (GPU time of the replays between CUDA events, and host wall time including the
spills), ms per step over the last 256 steps, the median and maximum spill time (host clock around the synchronising call), the
context's HBM bytes (mpig_device_bytes) and the device error flags.  The card's name and power limit are read in the same run.
Prints one JSON line.

    python scripts/shared_long_gen_bench.py [--B 8] [--N 4096] [--P 98000] [--M 131072] [--out FILE]
"""
import argparse
import gc
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner  # noqa: E402
from scripts.long_gen_bench import gpu_identity  # noqa: E402


def run_arm(args, gen_buf, spill):
    runner = LlamaDecodeRunner(LLAMA31_8B, args.K, args.L, args.B, args.M, generation_buffer=gen_buf, num_contexts=1,
                               dense_tail_rows=args.R, shared_spill=spill, num_layers=args.layers or None)
    runner.synthetic_prefill(args.P, shared=True)   # request 0 filled, forked to the others
    runner.ids.copy_(torch.arange(1, args.B + 1, device=runner.device)[:, None] * 1009)
    srv = runner.server
    used = runner.capture()                         # tokens the warm-up and the capture put into every window
    N = args.N
    start = [torch.cuda.Event(enable_timing=True) for _ in range(N)]
    end = [torch.cuda.Event(enable_timing=True) for _ in range(N)]
    spill_ms = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(N):
        if used == gen_buf:
            if not spill:
                raise RuntimeError("window full in the no-spill arm: raise its generation_buffer")
            torch.cuda.synchronize()                # the queued replays are not part of the spill
            ts = time.perf_counter()
            srv.spill_window()                      # synchronises
            spill_ms.append((time.perf_counter() - ts) * 1e3)
            used = 0
        start[i].record()
        runner.replay()
        end[i].record()
        used += 1
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    per = [a.elapsed_time(b) for a, b in zip(start, end)]
    tail = per[-256:]
    res = {
        "generation_buffer": gen_buf,
        "shared_spill": spill,
        "ms_per_step": sum(per) / N,
        "ms_per_step_last_256": sum(tail) / len(tail),
        "ms_per_step_wall": wall * 1e3 / N,
        "tokens_per_s": args.B * N / wall,
        "device_bytes": srv.ctx.device_bytes,
        "error_flags": srv.ctx.error_flags(),
        "spills": len(spill_ms),
    }
    if spill_ms:
        res["spill_ms_median"] = statistics.median(spill_ms)
        res["spill_ms_max"] = max(spill_ms)
    del runner, srv
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=8, help="requests forked from the prompt")
    ap.add_argument("--N", type=int, default=4096, help="generated tokens per request")
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--M", type=int, default=131072, help="max_length: the prompt plus every request's spilled tokens")
    ap.add_argument("--R", type=int, default=4400, help="dense_tail_rows: each request's dense rows after the prompt")
    ap.add_argument("--K", type=int, default=10)
    ap.add_argument("--L", type=int, default=150)
    ap.add_argument("--gen-buf", type=int, default=256, help="generation_buffer of the spilling arm")
    ap.add_argument("--layers", type=int, default=0, help="debug: fewer layers (the result is then not the workload)")
    ap.add_argument("--arms", default="ab")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("shared_long_gen_bench needs a CUDA device (H100); there is nothing to measure without one")
    line = {"metric": "shared_long_generation", "model": "llama-3.1-8b (synthetic weights)", "B": args.B, "contexts": 1,
            "P": args.P, "M": args.M, "R": args.R, "N": args.N, "K": args.K, "L": args.L, "gpu": gpu_identity()}
    if "a" in args.arms:
        line["arm_a_shared_spill"] = run_arm(args, args.gen_buf, spill=True)
    if "b" in args.arms:
        line["arm_b_no_spill"] = run_arm(args, args.N + 8, spill=False)   # the capture's warm-up tokens also occupy the window
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
