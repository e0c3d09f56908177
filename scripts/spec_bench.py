"""Speculative decoding on the H100: the acceptance kernel (mpig_aux_verify_sample) next to mpig_aux_sample and next to the same rule
in eager torch ops, the prompt-lookup drafter (mpig_aux_ngram_draft) at a 99 024-token history, the captured spec_step graph at the
bench shape, and generate() of 1 024 tokens from a 98 000-token prompt with k = 0, 1, 3, 7 drafts.  Writes
profiles/h100_spec_line.json (or --out) with the card's name, power limit and max SM clock read in the same run.

  verify     µs per call at B = 1, 8, 32, T = 1, 2, 4, 8, V = 128 256, greedy and T = 0.6 / top_p = 0.9: 50 calls captured in one
             graph, replayed 20 times between CUDA events (sample_bench.graph_us).  `sample_us`: mpig_aux_sample on the same B rows.
             `torch_eager_us`: the rule as a host-side caller would write it with torch ops (softmax, sort, cumsum, nucleus mask,
             acceptance of each draft, the residual and a multinomial draw), launched eagerly.
  ngram      µs per call at n = 99 024, B = 1 and 8, same graph timing.
  spec_step  the captured spec_step(k + 1) on a synthetic 98 000-token context (Llama-3.1-8B shapes, K10 L150, B = 1) against the
             captured step(), alternated blocks of replays, ms per replay.
  generate   generate() of --new tokens (no EOS ids, T = 0.6, top_p = 0.9) from a --P-token prompt of seeded random ids with
             draft_tokens = 0, 1, 3, 7: decode tokens/s, mean tokens per step, the spills (host clock, synchronised).

  python scripts/spec_bench.py [--out profiles/h100_spec_line.json] [--P 98000] [--new 1024] [--layers 32]
"""
import argparse
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
from sample_bench import eager_us, graph_us  # noqa: E402
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner  # noqa: E402
from magicpig_b200.ops import ngram_draft, sample, verify_sample  # noqa: E402

DEV = "cuda:0"
V = 128256


def torch_verify(logits, ids, temperature, top_p):
    """The speculative-sampling rule in torch ops, as a host-side caller writes it: logits (B, T, V), drafts ids[:, 1:T]."""
    B, T, _ = logits.shape
    if temperature <= 0:
        am = logits.argmax(-1)
        ok = (am[:, :T - 1] == ids[:, 1:T]).int()
        k = torch.cumprod(ok, 1).sum(1)
        return am.gather(1, k[:, None])[:, 0], T - 1 - k
    probs = torch.softmax(logits / temperature, dim=-1)
    sp, si = torch.sort(probs, dim=-1, descending=True)
    drop = torch.cumsum(sp, dim=-1) - sp > top_p
    sp = sp.masked_fill(drop, 0.0)
    q = torch.zeros_like(probs).scatter_(-1, si, sp)
    q = q / q.sum(-1, keepdim=True)
    d = ids[:, 1:T]
    pd = q[:, :T - 1].gather(-1, d[..., None])[..., 0]
    ok = (torch.rand(pd.shape, device=pd.device) < pd).int()
    k = torch.cumprod(ok, 1).sum(1)
    rows = q[torch.arange(B, device=q.device), k]
    dk = torch.cat([d, torch.zeros((B, 1), dtype=d.dtype, device=d.device)], 1).gather(1, k[:, None])
    res = rows.scatter(-1, dk, 0.0) * (k < T - 1)[:, None] + rows * (k == T - 1)[:, None]
    return torch.multinomial(res, 1)[:, 0], T - 1 - k


def verify_lines():
    out = []
    for B in (1, 8, 32):
        g = torch.Generator(device=DEV).manual_seed(B)
        for T in (1, 2, 4, 8):
            logits = torch.randn((B, T, V), generator=g, device=DEV) * 3
            ids = torch.randint(0, V, (B, 8), generator=g, device=DEV)
            ids[:, 1:T] = logits[:, :T - 1].argmax(-1)   # drafts that are accepted often
            ids0 = ids.clone()
            off = torch.zeros(1, dtype=torch.int64, device=DEV)
            drop = torch.zeros(B, dtype=torch.int32, device=DEV)
            rows = torch.zeros((B, T, 2), dtype=torch.int32, device=DEV)
            for arm, temp, p in (("greedy", 0.0, 1.0), ("top_p_0.9", 0.6, 0.9)):
                Tt, pt = torch.full((B,), temp, device=DEV), torch.full((B,), p, device=DEV)

                def call():
                    ids.copy_(ids0)
                    verify_sample(logits, Tt, pt, 1, off, ids, rows=rows, drop=drop)
                ours = graph_us(call) - graph_us(lambda: ids.copy_(ids0))
                line = dict(B=B, T=T, V=V, arm=arm, verify_us=round(ours, 2))
                if T == 1:
                    line["sample_us"] = round(graph_us(lambda: sample(logits[:, 0], Tt, pt, 1, off)), 2)
                ref = eager_us(lambda: torch_verify(logits, ids0, temp, p))
                line.update(torch_eager_us=round(ref, 2), speedup=round(ref / ours, 1))
                out.append(line)
                print(json.dumps(line), flush=True)
    return out


def ngram_lines(n=99024):
    out = []
    for B in (1, 8):
        g = torch.Generator(device=DEV).manual_seed(B)
        hist = torch.randint(0, V, (B, n + 1024), generator=g, device=DEV, dtype=torch.int32)
        length = torch.full((B,), n, dtype=torch.int32, device=DEV)
        ids = torch.zeros((B, 8), dtype=torch.int64, device=DEV)
        for T in (2, 8):
            us = graph_us(lambda: ngram_draft(hist, length, ids, T))
            out.append(dict(B=B, n=n, T=T, ngram_us=round(us, 2)))
            print(json.dumps(out[-1]), flush=True)
    return out


def spec_step_lines(run, P, blocks=5, per=10):
    """Captured step() against captured spec_step(k + 1), alternated blocks; the context is re-made before each graph's capture and
    the window spilled between blocks."""
    srv = run.server
    res = {}
    run.capture()
    graphs = {"step": run.graph}
    hist, length, limit, done = run._history()
    length.fill_(P)
    limit.fill_(hist.shape[1])
    for k in (1, 3, 7):
        run.ngram = (1, 3)
        run.capture(warm=2, draft_tokens=k)
        graphs[f"spec_k{k}"] = run.graph
        srv.spill_window()
    run.set_sampling(0.6, 0.9, seed=0, offset=0)
    for _ in range(blocks):
        for name, gr in graphs.items():
            done.zero_()
            length.fill_(P)
            srv.spill_window()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(per):
                gr.replay()
            e1.record()
            torch.cuda.synchronize()
            res.setdefault(name, []).append(e0.elapsed_time(e1) / per)
    return {name: dict(ms=[round(x, 4) for x in v], ms_median=round(statistics.median(v), 4)) for name, v in res.items()}


def generate_line(run, P, n_new, k):
    t = {"spill": []}
    srv = run.server
    f = srv.spill_window

    def timed(*a, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = f(*a, **kw)
        torch.cuda.synchronize()
        t["spill"].append(time.perf_counter() - t0)
        return r
    srv.spill_window = timed
    orig = {name: getattr(run, name) for name in ("prefill", "capture", "synthetic_prefill")}
    setup = [0.0]

    def wrap(fn):
        def w(*a, **kw):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **kw)
            torch.cuda.synchronize()
            setup[0] += time.perf_counter() - t0
            return r
        return w
    for name, fn in orig.items():
        setattr(run, name, wrap(fn))
    ids = torch.randint(0, V, (P,), generator=torch.Generator(device=DEV).manual_seed(7), device=DEV)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = run.generate(ids, n_new, temperature=0.6, top_p=0.9, eos_token_ids=(), seed=1, draft_tokens=k)
    total = time.perf_counter() - t0
    for name, fn in orig.items():
        setattr(run, name, fn)
    srv.spill_window = f
    decode = total - setup[0]
    n = len(out[0])
    line = dict(draft_tokens=k, P=P, new_tokens=n, total_s=round(total, 3), prefill_and_capture_s=round(setup[0], 3),
                decode_s=round(decode, 3), decode_tokens_per_s=round(n / decode, 1), spills=len(t["spill"]),
                spill_ms_total=round(sum(t["spill"]) * 1e3, 2), first_tokens=out[0][:8])
    if k:
        st = run.last_generate_stats
        line.update(steps=st["steps"][0], accepted_drafts=st["accepted"][0], tokens_per_step=round(st["tokens_per_step"], 4))
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(HERE), "profiles", "h100_spec_line.json"))
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--new", type=int, default=1024)
    ap.add_argument("--layers", type=int, default=0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "spec_bench.py measures on a CUDA device"
    line = dict(card=card(), torch=torch.__version__)
    print(line, flush=True)
    line["verify"] = verify_lines()
    line["ngram"] = ngram_lines()
    M = args.P + args.new + 256
    run = LlamaDecodeRunner(LLAMA31_8B, 10, 150, 1, M, device=DEV, num_layers=args.layers or None, max_query_tokens=8)
    run.synthetic_prefill(args.P)
    line["spec_step"] = dict(P=args.P, K=10, L=150, B=1, **spec_step_lines(run, args.P))
    print(json.dumps(line["spec_step"]), flush=True)
    line["generate"] = []
    for k in (0, 1, 3, 7):
        line["generate"].append(generate_line(run, args.P, args.new, k))
        print(json.dumps(line["generate"][-1]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(line, f, indent=1)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
