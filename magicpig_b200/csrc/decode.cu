// decode.cu -- the per-layer decode entry points.
// Sparse layers: ONE launch of fused_decode_kernel (fused.cu: SimHash -> probe -> gather attention + window merge) wherever
// its shape rules allow (option "decode_impl" = 1, the default); otherwise, and for the per-stage timing entry point, three
// launches  simhash_kernel (+ window append) -> probe_kernel -> attend_mma_kernel  chained with programmatic dependent launch.
// Replaces LSHSparseAttnServer.decode (models/attnserver.py:228-312) for sparse layers and, when the
// context owns the dense KV (cfg.alloc_dense_kv), the dense branch (:235-259).
#include <atomic>

#include "common.cuh"


using namespace mpig;

static int decode_sparse(mpig_ctx *ctx, int layer, const void *q, const void *k, const void *v, void *out, cudaStream_t s,
                         cudaEvent_t *ev = nullptr) {
    if (!ev && fused_applicable(ctx)) return launch_fused(ctx, layer, q, k, v, out, s, true);
    ctx->last_decode_fused = 0;
    ctx->last_tokens = 1;
    ctx->last_chunk = false;
    const LayerStore &ls = ctx->layers[layer];
    const AppendParams ap = append_params(ctx, ls, k, v, false);
    const bool pdl = (ev == nullptr);
    if (ev) MPIG_CUDA(cudaEventRecord(ev[0], s));
    // PDL on the first kernel too: it may start (and prefetch its hash_func slice) while the caller's previous kernel drains;
    // it reads q / k / v only after griddepcontrol.wait
    int rc = launch_simhash(ctx, q, ctx->codes, ctx->qnorm, &ap, s, pdl && ctx->pdl_first);
    if (rc) return rc;
    if (ev) MPIG_CUDA(cudaEventRecord(ev[1], s));
    rc = launch_probe(ctx, layer, ctx->codes, ctx->results, ctx->nnz, s, pdl);
    if (rc) return rc;
    if (ev) MPIG_CUDA(cudaEventRecord(ev[2], s));
    AttendParams p = attend_params(ctx, q, ctx->qnorm, out);
    p.kv = ls.kv;
    p.kn = ls.kn;
    p.slot_of = ctx->slot_map();
    p.win = ls.win;
    p.win_len = ctx->win_len;
    p.ind = ctx->results;
    p.nnz = ctx->nnz;
    p.mve = ctx->mve;
    rc = launch_attend_mma(ctx, p, s, pdl);
    if (rc) return rc;
    if (ev) MPIG_CUDA(cudaEventRecord(ev[3], s));
    return MPIG_OK;
}

extern "C" {

int mpig_decode(mpig_ctx *ctx, int layer, const void *query_bf16, const void *key_bf16, const void *value_bf16, void *out_bf16,
                void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_decode");
    if (rc) return rc;
    MPIG_REQUIRE(query_bf16 && key_bf16 && value_bf16 && out_bf16, MPIG_EINVAL, "mpig_decode: null argument");
    return decode_sparse(ctx, layer, query_bf16, key_bf16, value_bf16, out_bf16, as_stream(stream));
}

int mpig_decode_timed(mpig_ctx *ctx, int layer, const void *query_bf16, const void *key_bf16, const void *value_bf16,
                      void *out_bf16, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_decode_timed");
    if (rc) return rc;
    MPIG_REQUIRE(query_bf16 && key_bf16 && value_bf16 && out_bf16, MPIG_EINVAL, "mpig_decode_timed: null argument");
    const size_t need = (size_t)(ctx->timing_calls + 1) * 4;
    while (ctx->timing_events.size() < need) {
        cudaEvent_t e;
        MPIG_CUDA(cudaEventCreate(&e));
        ctx->timing_events.push_back(e);
    }
    rc = decode_sparse(ctx, layer, query_bf16, key_bf16, value_bf16, out_bf16, as_stream(stream),
                       &ctx->timing_events[(size_t)ctx->timing_calls * 4]);
    if (rc) return rc;
    ctx->timing_calls++;
    return MPIG_OK;
}

int mpig_timing_collect(mpig_ctx *ctx, float *stage_ms, int max_calls, int *n_calls) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx && stage_ms && n_calls, MPIG_EINVAL, "mpig_timing_collect: null argument");
    const int n = ctx->timing_calls < max_calls ? ctx->timing_calls : max_calls;
    if (ctx->timing_calls > 0) MPIG_CUDA(cudaEventSynchronize(ctx->timing_events[(size_t)ctx->timing_calls * 4 - 1]));
    for (int c = 0; c < n; ++c)
        for (int i = 0; i < 3; ++i)
            MPIG_CUDA(cudaEventElapsedTime(&stage_ms[c * 3 + i], ctx->timing_events[(size_t)c * 4 + i],
                                           ctx->timing_events[(size_t)c * 4 + i + 1]));
    *n_calls = n;
    ctx->timing_calls = 0;
    return MPIG_OK;
}

int mpig_decode_host(mpig_ctx *ctx, int layer, const void *query_bf16, const void *key_bf16, const void *value_bf16,
                     void *out_bf16, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_decode_host");
    if (rc) return rc;
    MPIG_REQUIRE(query_bf16 && key_bf16 && value_bf16 && out_bf16, MPIG_EINVAL, "mpig_decode_host: null argument");
    cudaStream_t s = as_stream(stream);
    // The kernels read q/k/v from, and write the output to, ONE mapped pinned block directly (zero-copy over PCIe: 12 KB in,
    // 8 KB out at C2): no cudaMemcpyAsync calls at all.  With the fused kernel the host does not even synchronise the stream: each
    // head's leader raises a flag in the same mapped block once its output row is written (fence, then the flag) and the host spins
    // on the H flags.  (Round 1 issued three H2D copies, the kernels, one D2H copy and a stream synchronisation: 72 us per layer.)
    const size_t qb = (size_t)ctx->H * ctx->cfg.head_dim * 2, kb = (size_t)ctx->BG * ctx->cfg.head_dim * 2;
    const size_t flag_off = ((qb + 2 * kb + qb) + 255) & ~(size_t)255;
    uint8_t *hq = (uint8_t *)ctx->host_stage, *hk = hq + qb, *hv = hk + kb, *hout = hv + kb;
    uint8_t *dq = (uint8_t *)ctx->host_stage_dev, *dk = dq + qb, *dv = dk + kb, *dout = dv + kb;
    volatile uint32_t *hflags = reinterpret_cast<volatile uint32_t *>(hq + flag_off);
    volatile uint32_t *dflags = reinterpret_cast<volatile uint32_t *>(dq + flag_off);
    // The block is this call's alone: the previous call returned only after every head's flag was seen (or the stream was idle),
    // i.e. after the last read of q/k/v and the last write of the output.
    memcpy(hq, query_bf16, qb);
    memcpy(hk, key_bf16, kb);
    memcpy(hv, value_bf16, kb);
    if (fused_applicable(ctx)) {
        const uint32_t epoch = ++ctx->host_epoch;
        rc = launch_fused(ctx, layer, dq, dk, dv, dout, s, true, nullptr, 0, 1, dflags, epoch);
        if (rc) return rc;
        // spin on the flags; if the kernel died the stream reports it
        unsigned long long spins = 0;
        for (int h = 0; h < ctx->H; ++h) {
            while (hflags[h] != epoch) {
                if ((++spins & 0xfffff) == 0) {   // ~every few ms: is the stream still alive?
                    cudaError_t e = cudaStreamQuery(s);
                    if (e != cudaErrorNotReady) {
                        MPIG_CUDA(e);
                        if (hflags[h] == epoch) break;
                        MPIG_CUDA(cudaStreamSynchronize(s));
                        break;
                    }
                }
            }
        }
        std::atomic_thread_fence(std::memory_order_acquire);
    } else {
        rc = decode_sparse(ctx, layer, dq, dk, dv, dout, s);
        if (rc) return rc;
        MPIG_CUDA(cudaStreamSynchronize(s));
    }
    memcpy(out_bf16, hout, qb);
    return MPIG_OK;
}

int mpig_dense_fill(mpig_ctx *ctx, int layer, int request, const void *k_bf16, const void *v_bf16, int seq_len, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, false, "mpig_dense_fill");
    if (rc) return rc;
    const LayerStore &ls = ctx->layers[layer];
    MPIG_REQUIRE(ls.dense && ls.dense_kv, MPIG_ESTATE, "mpig_dense_fill: layer %d has no dense KV (alloc_dense_kv=0 or sparse layer)",
                 layer);
    MPIG_REQUIRE(request >= 0 && request < ctx->cfg.batch_size, MPIG_EINVAL, "mpig_dense_fill: request %d out of range", request);
    MPIG_REQUIRE(seq_len >= 0 && seq_len <= ctx->cfg.max_length, MPIG_EINVAL, "mpig_dense_fill: seq_len=%d exceeds max_length",
                 seq_len);
    const int Hkv = ctx->cfg.num_key_value_heads, M = ctx->cfg.max_length;
    // shared dense mode: the rows go to the slot the request is bound to (as the sparse fills), and they become its base
    const bool shared = ctx->dense_tail_rows > 0;
    rc = refresh_maps(ctx, as_stream(stream));
    if (rc) return rc;
    const size_t owner = shared ? (size_t)ctx->h_slot_of[request] : (size_t)request;
    uint4 *rec = reinterpret_cast<uint4 *>(ls.dense_kv + owner * Hkv * M * ctx->rec_bytes);
    if (seq_len > 0) {
        rc = launch_pack_nhd(ctx, k_bf16, v_bf16, (uint8_t *)rec, Hkv, seq_len, M, as_stream(stream));
        if (rc) return rc;
    }
    MPIG_CUDA(cudaMemcpyAsync(ctx->dense_len + request, &seq_len, sizeof(int), cudaMemcpyHostToDevice, as_stream(stream)));
    if (shared) MPIG_CUDA(cudaMemcpyAsync(ctx->dense_base + request, &seq_len, sizeof(int), cudaMemcpyHostToDevice, as_stream(stream)));
    MPIG_CUDA(cudaStreamSynchronize(as_stream(stream)));  // seq_len is a stack variable
    ctx->h_dense_len[request] = seq_len;
    if (shared) ctx->h_dense_base[request] = seq_len;
    return MPIG_OK;
}

// the body of the two dense entry points: append the T new rows, then attend over the layer's dense KV
static int dense_decode(mpig_ctx *ctx, int layer, int T, const void *q, const void *k, const void *v, void *out, cudaStream_t s,
                        const char *who) {
    const LayerStore &ls = ctx->layers[layer];
    MPIG_REQUIRE(ls.dense && ls.dense_kv, MPIG_ESTATE, "%s: layer %d has no dense KV", who, layer);
    if (ctx->dense_impl == 1) {
        MPIG_REQUIRE(T * ctx->G <= 32, MPIG_EUNSUPPORTED, "%s: T*G = %d query rows per kv-group (at most 32)", who, T * ctx->G);
    } else {
        MPIG_REQUIRE(T == 1, MPIG_EUNSUPPORTED, "%s: T=%d needs the GQA-shared dense kernel (dense_impl = 1)", who, T);
        MPIG_REQUIRE(ctx->dense_tail_rows == 0, MPIG_EUNSUPPORTED,
                     "%s: the shared dense layout (dense_tail_rows > 0) needs the GQA-shared dense kernel (dense_impl = 1)", who);
    }
    int rc = launch_append_tokens(ctx, append_params(ctx, ls, k, v, true), T, s, ctx->dense_base_map());
    if (rc) return rc;
    if (ctx->dense_impl == 1) return launch_attend_dense(ctx, ls, T, q, out, s, T > 1);
    // the cache as window rows; qnorm is unused by window rows but must be a valid pointer
    AttendParams p = attend_params(ctx, q, ctx->qnorm, out);
    p.win = ls.dense_kv;
    p.win_len = ctx->dense_len;
    p.Wcap = ctx->cfg.max_length;
    ctx->last_tokens = 1;
    ctx->last_chunk = false;
    return launch_attend_mma(ctx, p, s, false);
}

int mpig_dense_decode(mpig_ctx *ctx, int layer, const void *query_bf16, const void *key_bf16, const void *value_bf16,
                      void *out_bf16, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, false, "mpig_dense_decode");
    if (rc) return rc;
    MPIG_REQUIRE(query_bf16 && key_bf16 && value_bf16 && out_bf16, MPIG_EINVAL, "mpig_dense_decode: null argument");
    return dense_decode(ctx, layer, 1, query_bf16, key_bf16, value_bf16, out_bf16, as_stream(stream), "mpig_dense_decode");
}

// shared checks of the two T-token entry points
static int tokens_checks(mpig_ctx *ctx, int layer, int T, const void *q, const void *k, const void *v, const void *out, bool sparse,
                         const char *who) {
    int rc = check_layer(ctx, layer, sparse, who);
    if (rc) return rc;
    MPIG_REQUIRE(q && k && v && out, MPIG_EINVAL, "%s: null argument", who);
    MPIG_REQUIRE(T >= 1 && T <= ctx->tok_max, MPIG_EINVAL, "%s: T=%d outside [1, %d] (mpig_reserve_query_tokens sets the upper bound)",
                 who, T, ctx->tok_max);
    MPIG_REQUIRE(T == ctx->pending.T, MPIG_ESTATE, "%s: T=%d but the last plan was for %d token(s)", who, T, ctx->pending.T);
    MPIG_REQUIRE(!ctx->pending.chunk, MPIG_ESTATE, "%s: the pending step is a chunk step (mpig_plan_chunk): decode it with mpig_chunk_attend",
                 who);
    return MPIG_OK;
}

int mpig_decode_tokens(mpig_ctx *ctx, int layer, int T, const void *query_bf16, const void *key_bf16, const void *value_bf16,
                       void *out_bf16, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    int rc = tokens_checks(ctx, layer, T, query_bf16, key_bf16, value_bf16, out_bf16, true, "mpig_decode_tokens");
    if (rc) return rc;
    if (T == 1) return mpig_decode(ctx, layer, query_bf16, key_bf16, value_bf16, out_bf16, stream);
    return launch_fused_tokens(ctx, layer, T, query_bf16, key_bf16, value_bf16, out_bf16, as_stream(stream));
}

int mpig_dense_decode_tokens(mpig_ctx *ctx, int layer, int T, const void *query_bf16, const void *key_bf16, const void *value_bf16,
                             void *out_bf16, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    int rc = tokens_checks(ctx, layer, T, query_bf16, key_bf16, value_bf16, out_bf16, false, "mpig_dense_decode_tokens");
    if (rc) return rc;
    return dense_decode(ctx, layer, T, query_bf16, key_bf16, value_bf16, out_bf16, as_stream(stream), "mpig_dense_decode_tokens");
}

int mpig_chunk_attend(mpig_ctx *ctx, int layer, int T, const void *query_bf16, const void *key_bf16, const void *value_bf16,
                      void *out_bf16, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    int rc = check_layer(ctx, layer, false, "mpig_chunk_attend");
    if (rc) return rc;
    MPIG_REQUIRE(query_bf16 && key_bf16 && value_bf16 && out_bf16, MPIG_EINVAL, "mpig_chunk_attend: null argument");
    MPIG_REQUIRE(T >= 1 && T <= ctx->chunk_max, MPIG_EINVAL,
                 "mpig_chunk_attend: T=%d outside [1, %d] (mpig_reserve_chunk_tokens sets the upper bound)", T, ctx->chunk_max);
    MPIG_REQUIRE(ctx->pending.chunk && T == ctx->pending.T, MPIG_ESTATE,
                 "mpig_chunk_attend: the pending step is not a chunk step of %d token(s) (mpig_plan_chunk)", T);
    const LayerStore &ls = ctx->layers[layer];
    MPIG_REQUIRE(ls.sparse || ls.dense_kv, MPIG_ESTATE, "mpig_chunk_attend: dense layer %d has no dense KV (alloc_dense_kv = 0)", layer);
    return launch_chunk_attend(ctx, layer, T, query_bf16, key_bf16, value_bf16, out_bf16, as_stream(stream));
}

}  // extern "C"
