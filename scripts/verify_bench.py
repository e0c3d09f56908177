"""Verification steps of T tokens at the bench shape (Llama-3.1-8B, P = 98 000, K10 L150, B = 1): ms per step for T in {1, 2, 4, 8}.

    python scripts/verify_bench.py [--out profiles/h100_verify_line.json]

For every T, two CUDA graphs replayed with the lengths kept in place (plan(T) -> layers -> rewind(T)):
  attention  the 32 attention layers alone (30 sparse through mpig_decode_tokens, 2 dense through mpig_dense_decode_tokens) on
             static q / k / v;
  model      LlamaDecodeRunner.step_tokens(T, drop=T): embedding, 32 layers, lm_head over the B*T rows.
and, in the same process, the captured single-token step() that bench.py measures.  Also per T: the cluster waves of the fused
kernel and the algorithmic bytes of one step (weights, dense-layer KV records, the sparse layers' window + sampled records, counted
from the nnz of an eager pass).  Sparse bytes grow with T; weights and dense KV do not.  step_T / step_1 (model) is the acceptance
length a speculative loop needs to break even.  Prints one JSON line; --out also writes it to a file.

--trees adds token-tree steps (plan_tree(T) -> layers -> accept(count = 0), so the lengths stay put) for a chain of 4 and of 8
nodes, a binary tree of depth 3 (T = 7) and a star of 1 + 7 nodes (T = 8), with the same attention / model fields as the chain
lines, plus the accept kernel alone (torch.profiler over graph replays) with a path of 7 nodes that moves 6 rows per layer and
kv-head, and with count = 0.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import gpu_identity  # noqa: E402
from magicpig_b200.llama_runner import LLAMA31_8B, LlamaDecodeRunner  # noqa: E402

REC = 512   # bytes of one K|V record (d = 128, bf16)


def replay_ms(graph, iters: int, reps: int) -> float:
    """Median over `reps` blocks of `iters` replays, device events around each block."""
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            graph.replay()
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1) / iters)
    return statistics.median(out)


def capture(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    torch.cuda.synchronize()
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=98000)
    ap.add_argument("--M", type=int, default=98304)
    ap.add_argument("--K", type=int, default=10)
    ap.add_argument("--L", type=int, default=150)
    ap.add_argument("--B", type=int, default=1)
    ap.add_argument("--tokens", default="1,2,4,8")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--trees", action="store_true", help="also time token-tree steps and the accept kernel")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("verify_bench.py measures on the GPU; no CUDA device found")
    Ts = [int(t) for t in args.tokens.split(",")]
    dev = "cuda:0"
    sh = LLAMA31_8B
    runner = LlamaDecodeRunner(sh, args.K, args.L, args.B, args.M, device=dev, seed=0, generation_buffer=256,
                               max_query_tokens=8 if args.trees else max(Ts))
    t0 = time.time()
    runner.synthetic_prefill(args.P, seed=100)
    prefill_s = time.time() - t0
    srv, ctx = runner.server, runner.server.ctx
    B, Hq, Hkv, d = args.B, sh.num_attention_heads, sh.num_key_value_heads, sh.head_dim
    nl = runner.n_layers
    sparse_layers = [l for l in range(nl) if l not in srv.dense_layers]
    weight_bytes = sum(t.numel() * t.element_size() for lw in runner.layers for t in lw.values()) + \
        runner.lm_head.numel() * runner.lm_head.element_size()
    g = torch.Generator(device=dev).manual_seed(5)
    results = []
    for T in Ts:
        q = torch.randn((B, Hq, T, d), generator=g, device=dev).bfloat16()
        k = torch.randn((B, Hkv, T, d), generator=g, device=dev).bfloat16()
        v = torch.randn((B, Hkv, T, d), generator=g, device=dev).bfloat16()
        drop = torch.full((B,), T, dtype=torch.int32, device=dev)

        # eager pass: the sampled rows of every sparse layer (nnz per virtual head) for the byte count
        srv.plan(T)
        sampled = 0
        for li in range(nl):
            srv.decode(q, k, v, li)
            if li in sparse_layers:
                nnz, _ = ctx.last_probe()
                sampled += int(nnz.sum())
        waves = ctx.get_info("tokens_cluster_waves") if T > 1 else ctx.get_info("fused_cluster_waves")
        srv.rewind(drop)
        w0 = srv.num_sink_tokens + srv.num_local_tokens   # window rows before the step (no token generated yet)
        window_rows = len(sparse_layers) * B * Hq * sum(w0 + t + 1 for t in range(T))
        dense_rows = len(srv.dense_layers) * B * Hkv * (args.P + T)

        def attention(T=T, q=q, k=k, v=v, drop=drop):
            srv.plan(T)
            for li in range(nl):
                srv.decode(q, k, v, li)
            srv.rewind(drop)

        ga = capture(attention)
        att_ms = replay_ms(ga, args.iters, args.reps)
        del ga
        runner.ids_tok.random_(0, sh.vocab_size, generator=g)
        gm = capture(lambda T=T, drop=drop: runner.step_tokens(T, drop))
        model_ms = replay_ms(gm, args.iters, args.reps)
        del gm
        results.append(dict(T=T, attention_ms=round(att_ms, 4), model_ms=round(model_ms, 4), cluster_waves=waves,
                            bytes=dict(weights=weight_bytes, dense_kv=dense_rows * REC, sparse_window=window_rows * REC,
                                       sparse_sampled=sampled * REC),
                            sparse_sampled_rows=sampled))
    trees = dict(per_tree=tree_lines(runner, args, g)) if args.trees else None
    # the single-token step bench.py measures, in the same process
    runner.capture()
    step1_ms = replay_ms(runner.graph, args.iters, args.reps)
    if trees:
        trees["accept"] = accept_lines(runner, args)   # last: it grows the lengths
    base = next((r for r in results if r["T"] == 1), None)
    for r in results + (trees["per_tree"] if trees else []):
        if base:
            r["break_even_accepted_tokens"] = round(r["model_ms"] / base["model_ms"], 3)
    line = dict(metric="verification step ms, Llama-3.1-8B @ P=98K, K10L150", B=B, P=args.P, K=args.K, L=args.L,
                captured_step_ms=round(step1_ms, 4), per_T=results, gpu=gpu_identity(0), prefill_s=round(prefill_s, 1),
                timing=f"CUDA events, median of {args.reps} blocks of {args.iters} graph replays")
    if trees:
        line.update(trees)
    text = json.dumps(line)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


TREES = {
    "chain4": [-1, 0, 1, 2],
    "chain8": [-1, 0, 1, 2, 3, 4, 5, 6],
    "binary_depth3": [-1, 0, 0, 1, 1, 2, 2],
    "star_1+7": [-1, 0, 0, 0, 0, 0, 0, 0],
}


def tree_lines(runner, args, g):
    """Tree steps with accept(count = 0): the lengths stay where they are."""
    srv, sh, dev = runner.server, runner.shape, runner.device
    B, Hq, Hkv, d = args.B, sh.num_attention_heads, sh.num_key_value_heads, sh.head_dim
    nl = runner.n_layers
    nodes0 = torch.zeros((B, 8), dtype=torch.int32, device=dev)
    count0 = torch.zeros((B,), dtype=torch.int32, device=dev)
    out = []
    for name, pars in TREES.items():
        T = len(pars)
        par = torch.tensor([pars] * B, dtype=torch.int32, device=dev)
        q = torch.randn((B, Hq, T, d), generator=g, device=dev).bfloat16()
        k = torch.randn((B, Hkv, T, d), generator=g, device=dev).bfloat16()
        v = torch.randn((B, Hkv, T, d), generator=g, device=dev).bfloat16()
        nodes = nodes0[:, :T].contiguous()

        def attention(T=T, par=par, q=q, k=k, v=v, nodes=nodes):
            srv.plan(T, parents=par)
            for li in range(nl):
                srv.decode(q, k, v, li)
            srv.accept(nodes, count0)

        ga = capture(attention)
        att_ms = replay_ms(ga, args.iters, args.reps)
        del ga
        runner.ids_tok.random_(0, sh.vocab_size, generator=g)
        gm = capture(lambda T=T, par=par, nodes=nodes: runner.step_tree(T, par, nodes, count0))
        model_ms = replay_ms(gm, args.iters, args.reps)
        del gm
        out.append(dict(tree=name, T=T, parents=pars, attention_ms=round(att_ms, 4), model_ms=round(model_ms, 4),
                        cluster_waves=srv.ctx.get_info("tokens_cluster_waves")))
    return out


def accept_lines(runner, args):
    """The accept kernel alone, from profiled graph replays of plan_tree(8) -> accept.  The moving path grows the lengths by 7 per
    replay, so this runs after every other measurement."""
    srv, sh, dev = runner.server, runner.shape, runner.device
    B, Hkv = args.B, sh.num_key_value_heads
    # the accept kernel alone: a comb tree whose path of 7 nodes moves 6 rows per (layer, request, kv-head), and count = 0
    comb = torch.tensor([[-1, 0, 0, 2, 3, 4, 5, 6]] * B, dtype=torch.int32, device=dev)
    path = torch.tensor([[0, 2, 3, 4, 5, 6, 7, 0]] * B, dtype=torch.int32, device=dev)
    accept = {}
    for label, cnt in (("path7_moves6", 7), ("count0", 0)):
        count = torch.full((B,), cnt, dtype=torch.int32, device=dev)
        srv.plan(8, parents=comb)
        srv.accept(path, count)   # eager warm-up
        gr = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s), torch.cuda.graph(gr, stream=s):
            srv.plan(8, parents=comb)
            srv.accept(path, count)
        torch.cuda.synchronize()
        reps = 8   # 8 x 7 rows of the 256-row generation buffer
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                gr.replay()
            torch.cuda.synchronize()
        us = [e.device_time_total for e in prof.events() if "accept_path_kernel" in e.name]
        accept[label] = dict(kernel_us_median=round(statistics.median(us), 2) if us else None, samples=len(us),
                             moved_bytes=runner.n_layers * B * Hkv * (6 if cnt else 0) * REC)
        del gr
    return accept


if __name__ == "__main__":
    main()
