"""Beam search over one shared context: what the device-side reorder (mpig_reorder_requests) costs per step.  Llama-3.1-8B shape
(synthetic weights, K = 10, L = 150), one context slot holding a P-token prompt with dense_tail_rows R, shared spill with
generation_buffer 256, B beams forked from the prompt.  Per beam width B:

  step_ms          the captured step() alone against the captured step() + beam_step (log_softmax, top-B over B x vocab,
                   beam_sources, reorder, token and score scatter) in one graph: blocks of replays between CUDA events, the two
                   graphs alternated block by block in one process, the median of the blocks' ms per step
  reorder_alone    a graph holding only the reorder with the worst-case map src_of = [0, 0, ..., 0] (B - 1 requests moved) at a
                   full window: ms per reorder, the bytes it moves (computed below from the lengths and the map) and the achieved
                   TB/s against the data sheet's 3.35 TB/s
  host_fork_ms     the same beam loop with the parents read to the host and one fork per moved beam, outside the graph (host
                   clock around steps that end in a synchronise)
  long_run         N tokens per beam of captured step() + beam_step, spilling every beam's window whenever it is full: GPU ms
                   per step (CUDA events around each replay), wall ms per step including the spills, spill count, error flags

The card's name and power limit are read in the same run.  Prints one JSON line.

    python scripts/beam_bench.py [--B 4 8] [--P 98000] [--N 1024] [--out FILE]
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
from magicpig_b200.attnserver import beam_sources  # noqa: E402
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner  # noqa: E402
from scripts.long_gen_bench import gpu_identity  # noqa: E402

REC = 512          # bytes of one K|V record (head_dim 128, bf16)
HBM_TBS = 3.35     # H100 SXM data sheet


def reorder_bytes(runner, src_of, win_rows, tail_rows):
    """bytes one reorder reads and writes: per moved request, every sparse layer's window rows and avg_k and every dense layer's
    tail rows for each kv-head, plus the visibility words of the shared spill map (read and written once)"""
    ctx = runner.server.ctx
    moved = sum(1 for b, s in enumerate(src_of) if s != b)
    n_dense = len(runner.server.dense_layers)
    n_sparse = runner.n_layers - n_dense
    per_req = ctx.Hkv * (n_sparse * (win_rows * REC + ctx.d * 2) + n_dense * tail_rows * REC)
    vis = ctx.C * ctx.M * 4 if ctx.shared_spill else 0
    return 2 * (moved * per_req + vis)


def timed_blocks(graph, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


class Beams:
    """A runner, its two graphs and the bookkeeping of the window rows and generated tokens since the prefill."""

    def __init__(self, args, B):
        self.args, self.B = args, B
        self.r = LlamaDecodeRunner(LLAMA31_8B, args.K, args.L, B, args.M, generation_buffer=args.gen_buf, num_contexts=1,
                                   dense_tail_rows=args.R, shared_spill=True)
        self.r.synthetic_prefill(args.P, shared=True)
        self.scores = torch.zeros(B, dtype=torch.float32, device=self.r.device)
        self.r.capture()
        self.g_step = self.r.graph
        self.r.capture(beam_scores=self.scores)
        self.g_beam = self.r.graph
        # window rows past sink + local, and tokens since the prefill: the two captures ran 3 warm-up steps each (a capture
        # itself runs nothing)
        self.used, self.tokens = 6, 6
        self.r.ids.fill_(1009)
        self.scores.copy_(torch.tensor([0.0] + [float("-inf")] * (B - 1)))

    def spill(self):
        torch.cuda.synchronize()
        t = time.perf_counter()
        self.r.server.spill_window()
        self.used = 0
        return (time.perf_counter() - t) * 1e3

    def room(self, n):
        if self.used + n > self.args.gen_buf:
            self.spill()

    def advance(self, n):
        self.used += n
        self.tokens += n


def measure(args, B):
    bm = Beams(args, B)
    r = bm.r
    # 1. step() against step() + beam_step, alternated block by block
    blk, arms = args.block, {"step": [], "step_beam": []}
    for _ in range(2):   # warm both graphs
        for g in (bm.g_step, bm.g_beam):
            bm.room(blk)
            timed_blocks(g, blk)
            bm.advance(blk)
    for _ in range(args.blocks):
        for name, g in (("step", bm.g_step), ("step_beam", bm.g_beam)):
            bm.room(blk)
            arms[name].append(timed_blocks(g, blk))
            bm.advance(blk)
    step_ms = {k: statistics.median(v) for k, v in arms.items()}
    step_ms["reorder_share_ms"] = step_ms["step_beam"] - step_ms["step"]
    step_ms["blocks"] = {k: v for k, v in arms.items()}

    # 2. the reorder alone at a full window, worst-case map
    bm.spill()
    for _ in range(args.gen_buf):
        bm.g_step.replay()
    bm.advance(args.gen_buf)
    torch.cuda.synchronize()
    win_rows = r.server.num_sink_tokens + r.server.num_local_tokens + args.gen_buf
    src = torch.zeros(B, dtype=torch.int32, device=r.device)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        r.reorder(src)   # eager once (the kernel is loaded)
    torch.cuda.synchronize()
    g_re = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g_re, stream=s):
            r.reorder(src)
    torch.cuda.synchronize()
    timed_blocks(g_re, 10)
    re_ms = statistics.median(timed_blocks(g_re, 50) for _ in range(5))
    nbytes = reorder_bytes(r, [0] * B, win_rows, bm.tokens)
    reorder = {"ms": re_ms, "moved": B - 1, "window_rows": win_rows, "dense_tail_rows_moved": bm.tokens, "bytes": nbytes,
               "tb_per_s": nbytes / (re_ms * 1e-3) / 1e12, "share_of_hbm_peak": nbytes / (re_ms * 1e-3) / 1e12 / HBM_TBS}
    bm.spill()

    # 3. the host alternative: parents to the host, one fork per moved beam, outside the graph
    host = []
    for i in range(args.host_steps):
        bm.room(1)
        torch.cuda.synchronize()
        t = time.perf_counter()
        bm.g_step.replay()
        parents, tokens, new = r.beam_select(bm.scores)
        src_of, request_of = beam_sources(parents)
        for dst, s_ in enumerate(src_of.tolist()):
            if s_ != dst:
                r.fork(s_, dst)
        r.ids[request_of.long(), 0] = tokens
        bm.scores[request_of.long()] = new
        torch.cuda.synchronize()
        host.append((time.perf_counter() - t) * 1e3)
        bm.advance(1)
    # the captured loop timed the same way (host clock, one step at a time)
    dev_loop = []
    for i in range(args.host_steps):
        bm.room(1)
        torch.cuda.synchronize()
        t = time.perf_counter()
        bm.g_beam.replay()
        torch.cuda.synchronize()
        dev_loop.append((time.perf_counter() - t) * 1e3)
        bm.advance(1)
    host_ms = {"host_forks_ms_per_step": statistics.median(host[2:]), "captured_beam_step_ms_per_step": statistics.median(dev_loop[2:])}

    # 4. a long run: N tokens per beam, spills included
    N = args.N
    starts = [torch.cuda.Event(enable_timing=True) for _ in range(N)]
    ends = [torch.cuda.Event(enable_timing=True) for _ in range(N)]
    spills = []
    bm.spill()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(N):
        if bm.used == args.gen_buf:
            spills.append(bm.spill())
        starts[i].record()
        bm.g_beam.replay()
        ends[i].record()
        bm.advance(1)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    per = [a.elapsed_time(b) for a, b in zip(starts, ends)]
    long_run = {"N": N, "ms_per_step": sum(per) / N, "ms_per_step_wall": wall * 1e3 / N, "spills": len(spills),
                "spill_ms_median": statistics.median(spills) if spills else None, "error_flags": r.server.ctx.error_flags(),
                "scores_finite": bool(torch.isfinite(bm.scores).all())}
    res = {"B": B, "step_ms": step_ms, "reorder_alone": reorder, "host_alternative": host_ms, "long_run": long_run,
           "device_bytes": r.server.ctx.device_bytes}
    del bm, r
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, nargs="+", default=[4, 8], help="beam widths")
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--M", type=int, default=0, help="max_length (0: P + every beam's spilled tokens)")
    ap.add_argument("--R", type=int, default=0, help="dense_tail_rows (0: enough for every step of the run)")
    ap.add_argument("--K", type=int, default=10)
    ap.add_argument("--L", type=int, default=150)
    ap.add_argument("--gen-buf", type=int, default=256)
    ap.add_argument("--N", type=int, default=1024, help="tokens per beam of the long run")
    ap.add_argument("--block", type=int, default=16, help="replays per timed block")
    ap.add_argument("--blocks", type=int, default=8, help="timed blocks per arm")
    ap.add_argument("--host-steps", type=int, default=24)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("beam_bench needs a CUDA device (H100); there is nothing to measure without one")
    steps = 6 + 4 * args.block * (2 + args.blocks) + args.gen_buf + 2 * args.host_steps + args.N + 64
    args.R = args.R or steps
    args.M = args.M or args.P + max(args.B) * steps + 1024
    line = {"metric": "beam_search_reorder", "model": "llama-3.1-8b (synthetic weights)", "contexts": 1, "P": args.P, "M": args.M,
            "R": args.R, "K": args.K, "L": args.L, "generation_buffer": args.gen_buf, "gpu": gpu_identity(), "widths": []}
    for B in args.B:
        line["widths"].append(measure(args, B))
    line["gpu_after"] = gpu_identity()
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
