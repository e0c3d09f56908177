"""Prefill on the H100: the prefill attention kernel alone (mpig_prefill_attend) next to the chunk-step kernel and torch SDPA measured
in the same run, and LlamaDecodeRunner.prefill of a whole prompt end to end (time to first-token logits).

Shape: Llama-3.1-8B (Hq/Hkv = 32/8, d = 128).  Kernel shapes (q_len, kv_len): (8 192, 8 192), (7 888, 98 000) (the last reference chunk
of a 98 000-token prompt), (98 000, 98 000) in one call, and the 12 chunks of a 98 000-token prompt in sequence.  Rates count
4*d*Hq FLOP per visible (query row, key); the share of peak is against the data sheet's 989 TFLOP/s dense BF16.  Writes
profiles/h100_prefill_line.json (or --out) with the card's name, power limit and max SM clock read in the same run.

  python scripts/prefill_bench.py [--out profiles/h100_prefill_line.json] [--P 98000] [--layers 32]
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from chunk_bench import card, kernel_lines  # noqa: E402
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner, plan_prefill_chunks  # noqa: E402
from magicpig_b200.ops import Context  # noqa: E402

DEV = "cuda:0"
PEAK_TFLOPS = 989.0   # H100 SXM data sheet: dense BF16
Hq, Hkv, d = 32, 8, 128


def flop(q_len, kv_len):
    """4*d*Hq per visible (row, key): query i sees kv_len - q_len + i + 1 keys."""
    return 4 * d * Hq * (q_len * (kv_len - q_len) + q_len * (q_len + 1) / 2)


def timed(fn, reps):
    fn()   # warm-up
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def line(name, ms, fl):
    tf = fl / ms / 1e9
    return dict(kernel=name, ms=round(ms, 3), tflops=round(tf, 1), share_of_peak=round(tf / PEAK_TFLOPS, 3))


def prefill_kernel_lines(P):
    ctx = Context(10, 150, 1, Hq, Hkv, d, 1, 1024, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(1)
    q = torch.randn((P, Hq, d), generator=g, device=DEV).bfloat16()
    k = torch.randn((P, Hkv, d), generator=g, device=DEV).bfloat16()
    v = torch.randn((P, Hkv, d), generator=g, device=DEV).bfloat16()
    out = torch.empty_like(q)
    lines = []
    for q_len, kv_len, reps in ((8192, 8192, 50), (7888, P, 10), (P, P, 3)):
        ms = timed(lambda: ctx.prefill_attend(q[kv_len - q_len:kv_len], k[:kv_len], v[:kv_len], out[:q_len]), reps)
        lines.append(dict(q_len=q_len, kv_len=kv_len, **line("attend_prefill_kernel", ms, flop(q_len, kv_len))))
        print(json.dumps(lines[-1]), flush=True)
    chunks = plan_prefill_chunks(P, 8192, 4, 64, P)
    ms = timed(lambda: [ctx.prefill_attend(q[a:b], k[:b], v[:b], out[a:b]) for a, b in chunks], 3)
    lines.append(dict(q_len=P, kv_len=P, chunks=len(chunks), **line("attend_prefill_kernel, 8192-token chunks", ms,
                                                                       sum(flop(b - a, b) for a, b in chunks))))
    print(json.dumps(lines[-1]), flush=True)
    ctx.close()
    return lines, (q, k, v)


def sdpa_lines(qkv, lens):
    """torch SDPA (is_causal, enable_gqa) at q_len = kv_len, where its top-left causal alignment equals bottom-right; the backend
    is the first of flash / memory-efficient / cuDNN that accepts the call (the math backend would materialise the scores)."""
    from torch.nn.attention import SDPBackend, sdpa_kernel
    q, k, v = qkv
    lines = []
    for n in lens:
        qt, kt, vt = (x[:n].transpose(0, 1)[None] for x in (q, k, v))
        for be in (SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION, SDPBackend.CUDNN_ATTENTION):
            try:
                with sdpa_kernel([be]):
                    ms = timed(lambda: F.scaled_dot_product_attention(qt, kt, vt, is_causal=True, enable_gqa=True), 3 if n > 10000 else 20)
            except RuntimeError as e:
                lines.append(dict(q_len=n, kv_len=n, backend=be.name, refused=str(e).splitlines()[0][:160]))
                continue
            lines.append(dict(q_len=n, kv_len=n, backend=be.name, **line("torch sdpa", ms, flop(n, n))))
            break
        print(json.dumps(lines[-1]), flush=True)
    return lines


def end_to_end(P, layers):
    run = LlamaDecodeRunner(LLAMA31_8B, 10, 150, 1, P + 512, device=DEV, seed=0, generation_buffer=256, num_layers=layers)
    g = torch.Generator(device=DEV).manual_seed(3)
    ids = torch.randint(0, LLAMA31_8B.vocab_size, (P,), generator=g, device=DEV)
    run.prefill(ids[:8300])   # warm-up: modules, library GEMM choices at the chunk shapes
    srv = run.server
    inner = srv.prefill_attention
    evs = []

    def attention(*a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        o = inner(*a, **kw)
        e1.record()
        evs.append((e0, e1))
        return o

    srv.prefill_attention = attention
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run.prefill(ids)   # ends with a device synchronise
    wall = time.perf_counter() - t0
    srv.prefill_attention = inner
    attn_s = sum(a.elapsed_time(b) for a, b in evs) / 1e3
    logits_ok = bool(torch.isfinite(run.logits).all())
    run.ids.fill_(int(run.logits[0].argmax()))
    run.capture()
    step_ms = timed(run.replay, 20)
    return dict(P=P, layers=layers, B=1, ttft_s=round(wall, 3), prompt_tok_per_s=round(P / wall, 1),
                attention_s=round(attn_s, 3), attention_share=round(attn_s / wall, 3), attention_calls=len(evs),
                step_ms=round(step_ms, 3), logits_finite=logits_ok, error_flags=srv.ctx.error_flags())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_prefill_line.json")
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--layers", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prefill_bench needs a GPU")
    res = dict(card=card(), card_fields="name, power.limit, clocks.max.sm", shape="Llama-3.1-8B Hq 32 Hkv 8 d 128",
               flop_rule="4*d*Hq per visible (query row, key)", peak_tflops=PEAK_TFLOPS)
    res["prefill_kernel"], qkv = prefill_kernel_lines(a.P)
    res["chunk_kernel"] = kernel_lines(1, a.P, False, (1024,))   # B = 1, T = 1 024 after P keys: the sparse and the dense layer
    res["sdpa"] = sdpa_lines(qkv, (8192, a.P))
    del qkv
    torch.cuda.empty_cache()
    chunk_tf = max(x["tflops"] for x in res["chunk_kernel"])
    res["rate_vs_chunk_kernel"] = {f'{x["q_len"]}x{x["kv_len"]}' + (" chunks" if "chunks" in x else ""): round(x["tflops"] / chunk_tf, 2)
                                   for x in res["prefill_kernel"]}
    res["end_to_end"] = end_to_end(a.P, a.layers)
    print(json.dumps(res["end_to_end"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(dict(card=res["card"], rate_vs_chunk_kernel=res["rate_vs_chunk_kernel"])))


if __name__ == "__main__":
    main()
