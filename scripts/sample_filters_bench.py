"""Sampling filters on the H100: mpig_aux_sample_filtered and mpig_aux_verify_sample_filtered next to the unfiltered calls and next to
the same processing in torch ops, and the captured generate() with and without filters.  Writes
profiles/h100_sample_filters_line.json (or --out) with the card's name, power limit and max SM clock read in the same run.

  calls     µs per call at V = 128 256, B = 1, 8, 32 and T = 1 (sample) or 1, 4, 8 (verify_sample), temperature 0.6, top_p 0.9, a
            table with 2 000 prompt tokens and 500 counted ones per request, in the variants: unfiltered, each filter alone
            (top_k 50, min_p 0.05, repetition_penalty 1.2, presence_penalty 0.5, frequency_penalty 0.5), all five, and `torch`: the
            penalties, top-k, top-p and min-p in eager torch ops followed by the unfiltered kernel on the processed logits (what a
            caller without the filtered calls would run; the verification rows' draft counts are not modelled there).  50 calls
            captured in one graph, replayed 20 times between CUDA events (sample_bench.graph_us); torch eagerly (eager_us).
  generate  generate() of --new tokens from a --P-token prompt of seeded random ids (Llama-3.1-8B shapes, K10 L150, B = 1, T = 0.6,
            top_p = 0.9, no EOS ids) with draft_tokens = 0 and 3, without filters and with all five: decode tokens/s.

  python scripts/sample_filters_bench.py [--out profiles/h100_sample_filters_line.json] [--P 98000] [--new 1024] [--layers 32]
"""
import argparse
import functools
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from chunk_bench import card  # noqa: E402
from sample_bench import eager_us, graph_us  # noqa: E402
from spec_bench import generate_line  # noqa: E402
from magicpig_b200 import ops  # noqa: E402
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner  # noqa: E402
from magicpig_b200.ops import SampleFilters, sample, verify_sample  # noqa: E402

DEV = "cuda:0"
V = 128256
ALONE = dict(top_k=50, min_p=0.05, repetition_penalty=1.2, presence_penalty=0.5, frequency_penalty=0.5)


def make_filters(B, g, **vals):
    f = SampleFilters.neutral(B, V, DEV)
    for name, v in vals.items():
        getattr(f, name).fill_(v)
    for b in range(B):
        f.table[b, torch.randint(0, V, (2000,), generator=g, device=DEV)] = ops.PROMPT_BIT
        f.table[b, torch.randint(0, V, (500,), generator=g, device=DEV)] += 1
    return f


def torch_filters(logits, f, temperature, top_k, top_p, min_p):
    """The five filters in torch ops on (rows, V) logits, Hugging Face's order; returns processed logits (-inf outside)."""
    e = f.table[:, :V].long() & 0xFFFFFFFF
    c = (e & 0x7FFFFFFF).float()
    seen = (e >> 31).bool() | (c > 0)
    r = f.repetition_penalty[:, None]
    l = torch.where(seen, torch.where(logits > 0, logits / r, logits * r), logits)
    l = l - f.frequency_penalty[:, None] * c - f.presence_penalty[:, None] * (c > 0).float()
    probs = torch.softmax(l / temperature, -1)
    sp, si = torch.sort(probs, -1, descending=True)
    keep = (torch.arange(V, device=logits.device)[None] < top_k).expand(logits.shape[0], V).clone()
    sk = sp * keep
    sk = sk / sk.sum(-1, keepdim=True)
    keep &= (torch.cumsum(sk, -1) - sk) <= top_p
    keep &= sp >= min_p * sp[:, :1]
    mask = torch.zeros_like(keep).scatter_(-1, si, keep)
    return l.masked_fill(~mask, float("-inf"))


def call_lines():
    out = []
    for B in (1, 8, 32):
        g = torch.Generator(device=DEV).manual_seed(B)
        for T in (1, 4, 8):
            logits = torch.randn((B, T, V), generator=g, device=DEV) * 3
            ids = torch.randint(0, V, (B, 8), generator=g, device=DEV)
            ids[:, 1:T] = logits[:, :T - 1].argmax(-1)
            ids0 = ids.clone()
            off = torch.zeros(1, dtype=torch.int64, device=DEV)
            Tt, pt = torch.full((B,), 0.6, device=DEV), torch.full((B,), 0.9, device=DEV)
            variants = {"unfiltered": None, **{k: make_filters(B, g, **{k: v}) for k, v in ALONE.items()},
                        "all": make_filters(B, g, **ALONE)}
            line = dict(B=B, T=T)
            for name, f in variants.items():
                if T == 1:
                    line[f"sample_{name}_us"] = round(graph_us(lambda: sample(logits[:, 0], Tt, pt, 1, off, filters=f)), 2)

                def vcall():
                    ids.copy_(ids0)
                    verify_sample(logits, Tt, pt, 1, off, ids, filters=f)
                line[f"verify_{name}_us"] = round(graph_us(vcall), 2)
            fa = variants["all"]
            rows = logits.reshape(B * T, V)
            ft = SampleFilters(*(x.repeat_interleave(T, 0) for x in (fa.top_k, fa.min_p, fa.repetition_penalty, fa.presence_penalty,
                                                                      fa.frequency_penalty, fa.table)))
            Tr, pr = Tt.repeat_interleave(T), pt.repeat_interleave(T)
            ones = torch.ones_like(pr)

            def tcall():
                proc = torch_filters(rows, ft, 0.6, ALONE["top_k"], 0.9, ALONE["min_p"])
                sample(proc, Tr, ones, 1, off)
            line["torch_all_us"] = round(eager_us(tcall), 2)
            out.append(line)
            print(json.dumps(line), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(HERE), "profiles", "h100_sample_filters_line.json"))
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--new", type=int, default=1024)
    ap.add_argument("--layers", type=int, default=0)
    ap.add_argument("--skip-generate", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "sample_filters_bench.py measures on a CUDA device"
    line = dict(card=card(), torch=torch.__version__)
    print(line, flush=True)
    line["calls"] = call_lines()
    line["generate"] = []
    if not args.skip_generate:
        M = args.P + args.new + 256
        run = LlamaDecodeRunner(LLAMA31_8B, 10, 150, 1, M, device=DEV, num_layers=args.layers or None, max_query_tokens=8)
        gen = run.generate
        for k in (0, 3):
            for filt in (False, True):
                run.generate = functools.partial(gen, **ALONE) if filt else gen
                res = dict(filters=filt, **generate_line(run, args.P, args.new, k))
                line["generate"].append(res)
                print(json.dumps(res), flush=True)
        run.generate = gen
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(line, f, indent=1)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
