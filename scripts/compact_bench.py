"""Compaction of a shared context (mpig_compact_context): what it reclaims, what it costs, and how far a generation gets with it.
Llama-3.1-8B shape (synthetic weights, K = 10, L = 150), one context slot holding a P-token prompt, B requests forked from it,
shared spill, dense_tail_rows R, max_length M, generation_buffer 256, one captured step.  Two workloads:

  churn   question churn: every 1024 tokens requests 1..B-1 are forked again from request 0, which kills the keys they spilled
          since the last fork; the dead count is known exactly (checked against what compact() returns)
  beam    beam search of width B: the captured step() + beam_step; how many lineages survive a window is whatever the random
          weights give, and is reported

Each workload runs twice from a fresh prefill: without compaction, and with a compaction after each spill; both arms run until
spill_window() is refused for capacity (or --N tokens per request, 0 = no cap).  Per compaction: keys reclaimed and still live,
the wall time of compact() (host clock around the synchronising call), the spill's wall time, and the mean GPU time of the
captured step over the 256 steps before and after it (CUDA events around each replay).  Per arm: the tokens per request reached.
The first --profile compactions that reclaim keys run again under torch.profiler (their wall times, marked "profiled", include
its overhead): GPU time per kernel and host time in the CUDA runtime calls of one compaction.  The card's name, power limit and
SM clock are read in the same run.  Prints one JSON line per workload.

    python scripts/compact_bench.py [--B 8] [--P 98000] [--M 131072] [--workloads churn beam] [--out FILE] [--append]
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicpig_b200 import _native as N  # noqa: E402
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner  # noqa: E402
from scripts.long_gen_bench import gpu_identity as card  # noqa: E402


def gpu_identity():
    """the card's name and power limit, and its current and maximum SM clocks"""
    ident = card()
    try:
        sm, sm_max = subprocess.check_output(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                                              "-i", "0"], text=True).strip().split(", ")
        ident.update(sm_clock_mhz=float(sm), sm_clock_max_mhz=float(sm_max))
    except (OSError, subprocess.CalledProcessError, ValueError):
        ident.update(sm_clock_mhz=None, sm_clock_max_mhz=None)
    return ident


KERNELS = ("compact_live", "compact_move", "compact_stage", "keyhash", "table_truncate", "table_merge")
RUNTIME = ("cudaMalloc", "cudaFree", "cudaStreamSynchronize", "cudaMemcpyAsync", "cudaLaunchKernel")


def profiled_compact(srv):
    """one compact() under torch.profiler: (reclaimed per slot, GPU ms per kernel family, host ms per CUDA runtime call)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        rec = srv.compact()
        torch.cuda.synchronize()
    gpu, host = {}, {}
    for e in prof.events():
        ms = (e.time_range.end - e.time_range.start) / 1e3
        if "CUDA" in str(e.device_type):
            key = next((k for k in KERNELS if k in e.name), "memcpy" if "emcpy" in e.name else "other")
            gpu[key] = gpu.get(key, 0.0) + ms
        else:
            key = next((k for k in RUNTIME if e.name.startswith(k)), None)
            if key:
                host[key] = host.get(key, 0.0) + ms
    return rec, gpu, host


def run_arm(args, workload, compact):
    B, gb = args.B, args.gen_buf
    r = LlamaDecodeRunner(LLAMA31_8B, args.K, args.L, B, args.M, generation_buffer=gb, num_contexts=1, dense_tail_rows=args.R,
                          shared_spill=True)
    scores = torch.zeros(B, dtype=torch.float32, device=r.device) if workload == "beam" else None
    r.synthetic_prefill(args.P, shared=True)
    r.capture(beam_scores=scores)
    r.server.clear()   # the warm-up steps moved the requests: start again from the prompt
    r.synthetic_prefill(args.P, shared=True)
    r.ids.fill_(1009)
    if scores is not None:
        scores.copy_(torch.tensor([0.0] + [float("-inf")] * (B - 1)))
    srv = r.server
    step_ms, events, compactions, spills = [], [], [], []
    since_fork = 0   # tokens each of requests 1..B-1 spilled since it was last forked (churn)
    expected_dead = 0
    used = tokens = 0
    refused = False
    limit = min(args.N or 10 ** 9, args.R - gb)   # the dense tails hold R rows past the prompt
    breakdown = []
    while tokens < limit:
        if used == gb:
            torch.cuda.synchronize()
            t = time.perf_counter()
            try:
                g = srv.spill_window()
            except N.MagicPigError as e:
                if "max_length" not in str(e):
                    raise
                refused = True
                break
            spills.append((time.perf_counter() - t) * 1e3)
            used = 0
            since_fork += int(g[1]) if workload == "churn" else 0
            if compact:
                # a churn compaction reclaims keys right after a re-fork, a beam compaction from the second on
                prof = len(breakdown) < args.profile and (expected_dead > 0 if workload == "churn" else len(compactions) > 0)
                t = time.perf_counter()
                if prof:
                    rec, gpu, host = profiled_compact(srv)
                    breakdown.append({"token": tokens, "reclaimed": int(rec[0]), "gpu_ms": gpu, "gpu_ms_total": sum(gpu.values()),
                                      "host_runtime_ms": host})
                else:
                    rec = srv.compact()
                ms = (time.perf_counter() - t) * 1e3
                rec = int(rec[0])
                compactions.append({"token": tokens, "reclaimed": rec, "live": srv.ctx.visibility()[0].ne(0).sum().item(),
                                    "compact_ms": ms, "profiled": prof, "spill_ms": spills[-1], "step": len(events)})
                if workload == "churn":
                    assert rec == expected_dead, (rec, expected_dead)
                    expected_dead = 0
        if workload == "churn" and tokens and tokens % 1024 == 0 and used == 0:
            # requests 1..B-1 were forked from 0 the last time: the keys they spilled since die now
            expected_dead = (B - 1) * since_fork
            for b in range(1, B):
                r.fork(0, b)
            since_fork = 0
        elif workload == "churn" and tokens == 0:
            expected_dead = 0
            for b in range(1, B):
                r.fork(0, b)
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r.replay()
        e.record()
        events.append((a, e))
        used += 1
        tokens += 1
    torch.cuda.synchronize()
    step_ms = [a.elapsed_time(e) for a, e in events]

    def mean(xs):
        return sum(xs) / len(xs) if xs else None

    for c in compactions:
        i = c.pop("step")
        c["step_ms_before"] = mean(step_ms[max(0, i - 256):i])
        c["step_ms_after"] = mean(step_ms[i:i + 256])
    res = {"compact": compact, "tokens_per_request": tokens, "refused_for_capacity": refused, "spills": len(spills),
           "spill_ms_mean": mean(spills), "step_ms_mean": mean(step_ms), "error_flags": srv.ctx.error_flags(),
           "compactions": compactions, "breakdown": breakdown}
    if scores is not None:
        res["scores_finite"] = bool(torch.isfinite(scores).all())
    del r, srv
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--M", type=int, default=131072)
    ap.add_argument("--R", type=int, default=0, help="dense_tail_rows (0: M - P + 256, every row the store could take)")
    ap.add_argument("--K", type=int, default=10)
    ap.add_argument("--L", type=int, default=150)
    ap.add_argument("--gen-buf", type=int, default=256)
    ap.add_argument("--N", type=int, default=0, help="cap on the tokens per request of an arm (0: until refused)")
    ap.add_argument("--profile", type=int, default=2, help="compactions that reclaim keys to run under torch.profiler")
    ap.add_argument("--workloads", nargs="+", default=["churn", "beam"])
    ap.add_argument("--out", default=None)
    ap.add_argument("--append", action="store_true", help="append the lines to --out instead of replacing it")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("compact_bench needs a CUDA device (H100); there is nothing to measure without one")
    args.R = args.R or args.M - args.P + 256
    lines = []
    for w in args.workloads:
        line = {"metric": "shared_context_compaction", "workload": w, "model": "llama-3.1-8b (synthetic weights)", "contexts": 1,
                "B": args.B, "P": args.P, "M": args.M, "R": args.R, "K": args.K, "L": args.L, "generation_buffer": args.gen_buf,
                "N": args.N, "gpu": gpu_identity()}
        line["without"] = run_arm(args, w, False)
        line["with"] = run_arm(args, w, True)
        line["gpu_after"] = gpu_identity()   # after the arms: the SM clock under load
        lines.append(json.dumps(line))
        print(lines[-1], flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a" if args.append else "w") as f:
            f.write("".join(s + "\n" for s in lines))


if __name__ == "__main__":
    main()
