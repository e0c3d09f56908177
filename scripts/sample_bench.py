"""Sampling on the H100: the sampler kernel (mpig_aux_sample) alone next to a torch sampler of the reference's algorithm on the same
logits, the captured decode step with and without sampling at the bench shape, and generate() of 1 024 tokens from a 98 000-token
prompt.  Writes profiles/h100_generate_line.json (or --out) with the card's name, power limit and max SM clock read in the same run.

  kernel     µs per call at B = 1, 8, 32 and V = 128 256 for greedy, T = 0.6 / top_p = 0.9 and T = 0.6 / top_p = 1.0: 50 calls
             captured in one CUDA graph, the graph replayed 20 times between CUDA events.  `torch_eager` is the reference's
             topp_temperature_decode algorithm (softmax, descending sort, cumsum, shifted mask, renormalise, multinomial, gather)
             written with torch ops and launched eagerly as the reference's caller runs it (argmax for the greedy arm), 200
             calls between CUDA events.
  step       the captured Llama-3.1-8B step (synthetic weights and context, B = 1, P = 98 000, K10 L150) against the captured
             step + sample, blocks of 20 replays alternated, ms per replay from CUDA events.
  generate   generate() of --new tokens (no EOS ids, T = 0.6, top_p = 0.9) from a --P-token prompt of seeded random ids: the
             prefill, the sampling graph's capture, the decode (tokens/s over the replays and spills) and the spills (host clock,
             synchronised), each timed by wrapping the runner's calls.

  python scripts/sample_bench.py [--out profiles/h100_generate_line.json] [--P 98000] [--new 1024] [--layers 32]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from chunk_bench import card  # noqa: E402
from magicpig_b200 import _native as N  # noqa: E402
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner  # noqa: E402
from magicpig_b200.ops import sample  # noqa: E402

DEV = "cuda:0"
V = 128256


def torch_topp(logits, temperature, top_p):
    """The reference's top-p / temperature sampler (models/utils.py) as torch ops, on (B, V) logits."""
    probs = torch.softmax(logits / temperature, dim=-1)
    sp, si = torch.sort(probs, dim=-1, descending=True)
    drop = torch.cumsum(sp, dim=-1) > top_p
    drop[:, 1:] = drop[:, :-1].clone()
    drop[:, 0] = False
    sp = sp.masked_fill(drop, 0.0)
    sp = sp / sp.sum(dim=-1, keepdim=True)
    return si.gather(-1, torch.multinomial(sp, 1))


def graph_us(fn, calls=50, reps=20):
    """µs per call: `calls` calls captured in one graph, replayed `reps` times between CUDA events."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * calls)


def eager_us(fn, calls=200):
    """µs per call of eager launches between CUDA events (the way the reference's caller runs its sampler)."""
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / calls


def kernel_lines():
    out = []
    c = ctypes.c_int(0)
    N.check(N.load().mpig_aux_sample_occupancy(V, ctypes.byref(c)), "mpig_aux_sample_occupancy")
    for B in (1, 8, 32):
        g = torch.Generator(device=DEV).manual_seed(B)
        logits = torch.randn((B, V), generator=g, device=DEV) * 3   # spread like a language model's logits
        off = torch.zeros(1, dtype=torch.int64, device=DEV)
        ids = torch.zeros((B, 1), dtype=torch.int64, device=DEV)
        for arm, T, p in (("greedy", 0.0, 1.0), ("top_p_0.9", 0.6, 0.9), ("top_p_1.0", 0.6, 1.0)):
            Tt = torch.full((B,), T, device=DEV)
            pt = torch.full((B,), p, device=DEV)
            ours = graph_us(lambda: sample(logits, Tt, pt, 1, off, ids_out=ids))
            ref = eager_us((lambda: torch_topp(logits, T, p)) if T > 0 else (lambda: logits.argmax(dim=-1)))
            out.append(dict(B=B, V=V, arm=arm, kernel_us=round(ours, 2), torch_eager_us=round(ref, 2), speedup=round(ref / ours, 1)))
            print(json.dumps(out[-1]), flush=True)
    return out, c.value


def step_lines(run, blocks=5, per=20):
    """Captured step against captured step + sample, alternated blocks of `per` replays.  Both graphs advance the context."""
    run.capture()
    g_step = run.graph
    run.capture(sample=True)
    g_samp = run.graph
    run.set_sampling(0.6, 0.9, seed=0, offset=0)
    res = {"step": [], "step_sample": []}
    for _ in range(blocks):
        for name, g in (("step", g_step), ("step_sample", g_samp)):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(per):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            res[name].append(e0.elapsed_time(e1) / per)
    med = {k: statistics.median(v) for k, v in res.items()}
    return dict(blocks=blocks, replays_per_block=per, step_ms=[round(x, 4) for x in res["step"]],
                step_sample_ms=[round(x, 4) for x in res["step_sample"]], step_ms_median=round(med["step"], 4),
                step_sample_ms_median=round(med["step_sample"], 4),
                sample_share=round((med["step_sample"] - med["step"]) / med["step"], 5))


def generate_line(run, P, n_new):
    """generate() with its phases timed by wrapping the runner's calls (host clock, synchronised)."""
    t = {"prefill": 0.0, "capture": 0.0, "spill": []}
    srv = run.server

    def wrap(obj, name, key):
        f = getattr(obj, name)

        def timed(*a, **kw):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = f(*a, **kw)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if key == "spill":
                t["spill"].append(dt)
            else:
                t[key] += dt
            return r
        setattr(obj, name, timed)

    wrap(run, "prefill", "prefill")
    wrap(run, "capture", "capture")
    wrap(run, "synthetic_prefill", "capture")
    wrap(srv, "spill_window", "spill")
    ids = torch.randint(0, V, (P,), generator=torch.Generator(device=DEV).manual_seed(7), device=DEV)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = run.generate(ids, n_new, temperature=0.6, top_p=0.9, eos_token_ids=(), seed=1)
    total = time.perf_counter() - t0
    decode = total - t["prefill"] - t["capture"]
    n = len(out[0])
    return dict(P=P, new_tokens=n, total_s=round(total, 3), prefill_s=round(t["prefill"], 3), capture_s=round(t["capture"], 3),
                decode_s=round(decode, 3), decode_tokens_per_s=round(n / decode, 1), spills=len(t["spill"]),
                spill_ms_total=round(sum(t["spill"]) * 1e3, 2),
                spill_ms_median=round(statistics.median(t["spill"]) * 1e3, 2) if t["spill"] else None,
                distinct_tokens=len(set(out[0])), first_tokens=out[0][:8])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(HERE), "profiles", "h100_generate_line.json"))
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--new", type=int, default=1024)
    ap.add_argument("--layers", type=int, default=0)
    ap.add_argument("--skip-kernel", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "sample_bench.py measures on a CUDA device"
    line = dict(card=card(), torch=torch.__version__)
    print(line, flush=True)
    if not args.skip_kernel:
        line["kernel"], line["resident_clusters_at_V"] = kernel_lines()
    M = args.P + args.new + 256
    run = LlamaDecodeRunner(LLAMA31_8B, 10, 150, 1, M, device=DEV, num_layers=args.layers or None)
    run.synthetic_prefill(args.P)
    line["step"] = dict(P=args.P, K=10, L=150, B=1, max_length=M, **step_lines(run))
    print(json.dumps(line["step"]), flush=True)
    line["generate"] = generate_line(run, args.P, args.new)
    print(json.dumps(line["generate"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(line, f, indent=1)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
