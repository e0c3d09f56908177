"""Batched decode over one context with a shared dense prefix (mpig_config.dense_tail_rows) -> one JSON line.

Llama-3.1-8B with random weights, a synthetic P-token context filled once (request 0) and forked, K10 L150, one context slot,
R = generation_buffer + t_max dense tail rows.  For every B: the captured step() time (CUDA events, median over blocks of
replays), aggregate tokens/s and the context's HBM bytes (B = 1 cannot share: it runs with R = 0).  Then at B = 8, R = 0 against
R > 0 (at --pair-P: two runners must fit at once), alternated block by block: the step times and the largest logit difference (the dense kernels sum in different orders).
Then the dense layers alone at B = 8 on a bare context of the same shape (two dense layers, Hq 32, Hkv 8): CUDA events around
plan + the two dense launches, with the bytes the algorithm reads (R = 0: every request's rows; R > 0: the prompt once per chunk
of requests plus every tail) and the achieved bytes/s.  The card's name and power limit are read in the same run.

    python scripts/shared_dense_bench.py --out profiles/h100_shared_dense_line.json
"""
import argparse
import gc
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicpig_b200 import synth  # noqa: E402
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner  # noqa: E402
from magicpig_b200.ops import Context  # noqa: E402
from scripts.shared_context_bench import card, median, time_block  # noqa: E402

DEV = "cuda:0"
T_MAX = 1


def make(B, R, P, M, K, L, gen):
    C = 1 if (R or B > 1) else None
    r = LlamaDecodeRunner(LLAMA31_8B, K, L, B, M, device=DEV, seed=0, generation_buffer=gen, num_contexts=C,
                          dense_tail_rows=R or None)
    r.synthetic_prefill(P, shared=True)
    r.ids.copy_(torch.arange(1, B + 1, device=DEV)[:, None] * 1009)
    r.capture()
    return r


def free():
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def dense_only(B, P, M, R, blocks, per_block):
    """Times plan + the two dense layers of a step at B requests over one slot, both layouts alternated."""
    Hq, Hkv, d = 32, 8, 128
    hf = synth.make_hash_func(d, 10, 150, seed=1)
    g = torch.Generator(device=DEV).manual_seed(3)
    ctxs = {}
    for r in (0, R):
        c = Context(10, 150, 2, Hq, Hkv, d, B, M, 4, 64, R + 64, dense_layers=[0, 1], alloc_dense_kv=True, device=DEV,
                    num_contexts=1, dense_tail_rows=r)
        c.set_hash_func(hf.to(DEV))
        for layer in (0, 1):
            k = torch.randn((P, Hkv, d), generator=g, device=DEV).bfloat16()
            c.dense_fill(layer, 0, k, k, P)
            del k
        for b in range(1, B):
            c.fork(0, b)
        ctxs[r] = c
    q = torch.randn((B, Hq, d), generator=g, device=DEV).bfloat16()
    k = torch.randn((B, Hkv, d), generator=g, device=DEV).bfloat16()
    out = torch.empty((B, Hq * d), dtype=torch.bfloat16, device=DEV)
    graphs = {}
    for r, c in ctxs.items():
        c.plan()
        c.dense_decode(0, q, k, k, out=out)
        c.dense_decode(1, q, k, k, out=out)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            for _ in range(per_block):
                c.dense_decode(0, q, k, k, out=out)
                c.dense_decode(1, q, k, k, out=out)
        graphs[r] = gr
    times = {r: [] for r in ctxs}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(blocks + 1):
        for r, gr in graphs.items():
            a.record()
            gr.replay()
            b.record()
            b.synchronize()
            times[r].append(a.elapsed_time(b) / per_block)
    rec, n = 512, P + 1
    bytes_ = {0: 2 * B * Hkv * n * rec, R: 2 * Hkv * (P + B) * rec}   # one chunk of 8 requests at G = 4, T = 1
    res = {}
    for r in ctxs:
        ms = median(times[r][1:])
        res[f"R={r}"] = {"dense_ms": round(ms, 4), "block_ms": [round(t, 4) for t in times[r][1:]], "bytes": bytes_[r],
                         "bytes_per_s": round(bytes_[r] / (ms * 1e-3), 1), "device_bytes": ctxs[r].device_bytes}
    del ctxs, graphs
    free()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--M", type=int, default=98304)
    ap.add_argument("--K", type=int, default=10)
    ap.add_argument("--L", type=int, default=150)
    ap.add_argument("--batches", default="1,2,4,8,16,32")
    ap.add_argument("--blocks", type=int, default=7)
    ap.add_argument("--per-block", type=int, default=20)
    ap.add_argument("--pair-P", type=int, default=49000, help="context of the R = 0 / R > 0 pair (two runners must fit at once)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device (an H100); nothing is measured without one")
    gen = 16 + args.blocks * args.per_block * 2 + 8   # window rows the warm-up, capture and replays use
    R = gen + T_MAX
    line = {"workload": f"Llama-3.1-8B random weights, synthetic shared context P={args.P}, K{args.K} L{args.L}, num_contexts=1, "
                        f"dense_tail_rows={R}", "card": card(), "runs": []}
    for B in [int(x) for x in args.batches.split(",")]:
        r = make(B, R if B > 1 else 0, args.P, args.M, args.K, args.L, gen)
        ctx = r.server.ctx
        for _ in range(10):
            r.replay()
        ms = median([time_block(r, args.per_block) for _ in range(args.blocks)])
        line["runs"].append({"B": B, "dense_tail_rows": ctx.dense_tail_rows, "step_ms": round(ms, 4),
                             "tokens_per_s": round(B * 1000.0 / ms, 1), "device_bytes": ctx.device_bytes})
        print(json.dumps(line["runs"][-1]), flush=True)
        del r, ctx
        free()
    bytes_by_b = {x["B"]: x["device_bytes"] for x in line["runs"] if x["dense_tail_rows"]}
    bs = sorted(bytes_by_b)
    if len(bs) > 1:
        line["device_bytes_per_added_request"] = round((bytes_by_b[bs[-1]] - bytes_by_b[bs[0]]) / (bs[-1] - bs[0]))
    # B = 8: R = 0 against R > 0, alternated
    Mp = ((args.pair_P + 64 + 1023) // 1024) * 1024
    runners = {r: make(8, r, args.pair_P, Mp, args.K, args.L, gen) for r in (0, R)}
    times = {r: [] for r in runners}
    for _ in range(10):
        for r in runners:
            runners[r].replay()
    diff = (runners[0].logits - runners[R].logits).abs().max().item()
    same_tok = torch.equal(runners[0].logits.argmax(-1), runners[R].logits.argmax(-1))
    for _ in range(args.blocks):
        for r in runners:
            times[r].append(time_block(runners[r], args.per_block))
        diff = max(diff, (runners[0].logits - runners[R].logits).abs().max().item())
        same_tok &= torch.equal(runners[0].logits.argmax(-1), runners[R].logits.argmax(-1))
    line["pair"] = {"B": 8, "P": args.pair_P, "M": Mp, "max_abs_logit_diff": diff, "argmax_equal": bool(same_tok),
                    "step_ms": {f"R={r}": round(median(times[r]), 4) for r in runners},
                    "block_ms": {f"R={r}": [round(t, 4) for t in times[r]] for r in runners},
                    "device_bytes": {f"R={r}": runners[r].server.ctx.device_bytes for r in runners}}
    print(json.dumps(line["pair"]), flush=True)
    del runners
    free()
    line["dense_layers_B8"] = dense_only(8, args.P, args.M, R, args.blocks, args.per_block)
    print(json.dumps(line["dense_layers_B8"]), flush=True)
    line["card_after"] = card()
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
