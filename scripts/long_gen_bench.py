"""Long generation past generation_buffer: the captured Llama-3.1-8B decode step (synthetic weights, B = 1, P = 98 000, K = 10,
L = 150) replayed for N generated tokens in two arms:

  a  generation_buffer = 256 (--gen-buf), spill_window() between replays whenever the window is full
  b  generation_buffer = N, no spill: the window becomes a dense attention over every generated token

Per arm: ms per token over the whole generation (GPU time of the replays between CUDA events, and host wall time including the
spills), ms per token over the last 256 tokens, and for arm a the median and maximum spill time (host clock around the
synchronising call).  The card's name and power limit are read in the same run.  Prints one JSON line.

    python scripts/long_gen_bench.py [--N 4096] [--P 98000] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner  # noqa: E402


def gpu_identity():
    try:
        name, limit = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                              text=True).strip().split(", ")
        return {"name": name, "power_limit_w": float(limit)}
    except (OSError, subprocess.CalledProcessError, ValueError):
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None}


def run_arm(args, M, gen_buf, spill):
    runner = LlamaDecodeRunner(LLAMA31_8B, args.K, args.L, 1, M, generation_buffer=gen_buf, num_layers=args.layers or None)
    runner.synthetic_prefill(args.P)
    srv = runner.server
    used = runner.capture()                    # tokens the warm-up and the capture put into the window
    N = args.N
    start = [torch.cuda.Event(enable_timing=True) for _ in range(N)]
    end = [torch.cuda.Event(enable_timing=True) for _ in range(N)]
    spill_ms = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(N):
        if used == gen_buf:
            if not spill:
                raise RuntimeError("window full in the no-spill arm: raise --gen-buf for arm b")
            torch.cuda.synchronize()           # the queued replays are not part of the spill
            ts = time.perf_counter()
            srv.spill_window()                 # synchronises
            spill_ms.append((time.perf_counter() - ts) * 1e3)
            used = 0
        start[i].record()
        runner.replay()
        end[i].record()
        used += 1
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    flags = srv.ctx.error_flags()
    per = [a.elapsed_time(b) for a, b in zip(start, end)]
    tail = per[-256:]
    res = {
        "generation_buffer": gen_buf,
        "ms_per_token": sum(per) / N,
        "ms_per_token_last_256": sum(tail) / len(tail),
        "ms_per_token_wall": wall * 1e3 / N,
        "error_flags": flags,
        "spills": len(spill_ms),
    }
    if spill_ms:
        res["spill_ms_median"] = statistics.median(spill_ms)
        res["spill_ms_max"] = max(spill_ms)
    del runner, srv
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=4096, help="generated tokens")
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--K", type=int, default=10)
    ap.add_argument("--L", type=int, default=150)
    ap.add_argument("--gen-buf", type=int, default=256, help="generation_buffer of the spilling arm")
    ap.add_argument("--layers", type=int, default=0, help="debug: fewer layers (the result is then not the workload)")
    ap.add_argument("--arms", default="ab")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("long_gen_bench needs a CUDA device (H100); there is nothing to measure without one")
    M = (args.P + args.N + 68 + 63) // 64 * 64
    line = {"metric": "long_generation", "model": "llama-3.1-8b (synthetic weights)", "B": 1, "P": args.P, "M": M, "N": args.N,
            "K": args.K, "L": args.L, "gpu": gpu_identity()}
    if "a" in args.arms:
        line["arm_a_spill"] = run_arm(args, M, args.gen_buf, spill=True)
    if "b" in args.arms:
        # the capture's warm-up tokens also occupy the window
        line["arm_b_no_spill"] = run_arm(args, M, args.N + 8, spill=False)
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
