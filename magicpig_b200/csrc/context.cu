// context.cu -- context lifetime, HBM allocation, options.
// Replaces LSH::alloc (lsh.cc:44-91), SparseAttentionServer::alloc (sparse_attention.cc:546-583),
// their clear()s (lsh.cc:293-306, sparse_attention.cc:586-598) and the buffer set-up of
// LSHSparseAttnServer.__init__ (attnserver.py:40-104).
#include <stdarg.h>

#include <algorithm>
#include <mutex>
#include <set>
#include <tuple>

#include "common.cuh"

// The layout of ABI version 1, byte for byte: a caller built against any header of that version keeps working.
static_assert(offsetof(mpig_config, alloc_dense_kv) == 120, "mpig_config layout");
static_assert(offsetof(mpig_config, ctas_per_sm) == 124, "mpig_config layout");
static_assert(offsetof(mpig_config, num_contexts) == 128, "mpig_config layout");
static_assert(offsetof(mpig_config, dense_tail_rows) == 132, "mpig_config layout");
static_assert(offsetof(mpig_config, shared_spill) == 136, "mpig_config layout");
static_assert(offsetof(mpig_config, reserved) == 140, "mpig_config layout");
static_assert(sizeof(mpig_config) == 156, "mpig_config layout");

namespace mpig {

int func_attr_once(const void *fn, cudaFuncAttribute attr, int value) {
    static std::mutex mu;
    static std::set<std::tuple<const void *, int, int, int>> done;  // (function, attribute, device, value)
    int dev = 0;
    MPIG_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(mu);
    const auto key = std::make_tuple(fn, (int)attr, dev, value);
    if (done.count(key)) return MPIG_OK;
    MPIG_CUDA(cudaFuncSetAttribute(fn, attr, value));
    done.insert(key);
    return MPIG_OK;
}

static thread_local char g_err[1024] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_layer(mpig_ctx *ctx, int layer, bool need_sparse, const char *who) {
    MPIG_REQUIRE(ctx != nullptr, MPIG_EINVAL, "%s: null context", who);
    MPIG_REQUIRE(layer >= 0 && layer < ctx->cfg.num_layers, MPIG_EINVAL, "%s: layer %d out of range [0,%d)", who,
                 layer, ctx->cfg.num_layers);
    if (need_sparse) {
        MPIG_REQUIRE(ctx->layers[layer].sparse, MPIG_ESTATE, "%s: layer %d is a dense layer (no tables / offload store)",
                     who, layer);
    }
    return MPIG_OK;
}

template <typename T>
static int dev_alloc(mpig_ctx *ctx, T **p, size_t bytes, bool zero = true) {
    if (bytes == 0) bytes = 16;
    cudaError_t e = cudaMalloc((void **)p, bytes);
    if (e != cudaSuccess) {
        set_error("cudaMalloc(%zu bytes) failed: %s (context already holds %zu bytes)", bytes, cudaGetErrorString(e),
                  ctx->bytes);
        (void)cudaGetLastError();
        return MPIG_ENOMEM;
    }
    ctx->bytes += bytes;
    if (zero) MPIG_CUDA(cudaMemset(*p, 0, bytes));
    return MPIG_OK;
}

__global__ void transpose_hash_func_kernel(const __nv_bfloat16 *__restrict__ src, __nv_bfloat16 *__restrict__ dst,
                                           int d, int KL) {
    // src (d, KL) -> dst (KL, d)
    int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= KL) return;
    for (int k = 0; k < d; ++k) dst[(size_t)col * d + k] = src[(size_t)k * KL + col];
}

}  // namespace mpig

using namespace mpig;

extern "C" {

const char *mpig_last_error(void) { return g_err; }
int mpig_abi_version(void) { return MPIG_ABI_VERSION; }

int mpig_create(const mpig_config *cfg, mpig_ctx **out) {
    MPIG_REQUIRE(cfg && out, MPIG_EINVAL, "mpig_create: null argument");
    *out = nullptr;
    MPIG_REQUIRE(cfg->abi_version == MPIG_ABI_VERSION, MPIG_EINVAL, "mpig_create: abi_version %d != %d",
                 cfg->abi_version, MPIG_ABI_VERSION);
    MPIG_REQUIRE(cfg->K >= 1 && cfg->K <= 15, MPIG_EINVAL, "mpig_create: K=%d outside [1,15]", cfg->K);
    MPIG_REQUIRE(cfg->L >= 1 && cfg->L <= 1024, MPIG_EINVAL, "mpig_create: L=%d outside [1,1024]", cfg->L);
    MPIG_REQUIRE(cfg->head_dim == 128, MPIG_EUNSUPPORTED, "mpig_create: head_dim=%d (only 128 is built)", cfg->head_dim);
    MPIG_REQUIRE(cfg->num_layers >= 1 && cfg->batch_size >= 1 && cfg->max_length >= 1, MPIG_EINVAL,
                 "mpig_create: num_layers/batch_size/max_length must be positive");
    MPIG_REQUIRE(cfg->num_key_value_heads >= 1 && cfg->num_attention_heads % cfg->num_key_value_heads == 0, MPIG_EINVAL,
                 "mpig_create: Hq=%d must be a multiple of Hkv=%d", cfg->num_attention_heads, cfg->num_key_value_heads);
    MPIG_REQUIRE(cfg->num_dense_layers >= 0 && cfg->num_dense_layers <= 16, MPIG_EINVAL, "mpig_create: num_dense_layers");
    MPIG_REQUIRE(cfg->num_sink_tokens >= 0 && cfg->num_local_tokens >= 0 && cfg->generation_buffer >= 0, MPIG_EINVAL,
                 "mpig_create: negative window size");
    MPIG_REQUIRE(cfg->ctas_per_sm >= 0 && cfg->ctas_per_sm <= 2, MPIG_EINVAL,
                 "mpig_create: ctas_per_sm = %d is not 0, 1 or 2", cfg->ctas_per_sm);
    MPIG_REQUIRE(cfg->num_contexts >= 0 && cfg->num_contexts <= cfg->batch_size, MPIG_EINVAL,
                 "mpig_create: num_contexts = %d outside [0, batch_size = %d]", cfg->num_contexts, cfg->batch_size);
    if (cfg->dense_tail_rows != 0) {   // shared dense mode: R tail rows per request, the prompt rows once per slot
        MPIG_REQUIRE(cfg->dense_tail_rows >= 1 && cfg->dense_tail_rows <= cfg->max_length, MPIG_EINVAL,
                     "mpig_create: dense_tail_rows = %d outside [1, max_length = %d]", cfg->dense_tail_rows, cfg->max_length);
        MPIG_REQUIRE(cfg->num_contexts > 0 && cfg->num_contexts < cfg->batch_size, MPIG_EINVAL,
                     "mpig_create: dense_tail_rows = %d needs fewer context slots than requests (num_contexts = %d, batch_size = %d)",
                     cfg->dense_tail_rows, cfg->num_contexts, cfg->batch_size);
        MPIG_REQUIRE(cfg->alloc_dense_kv, MPIG_EINVAL,
                     "mpig_create: dense_tail_rows = %d needs alloc_dense_kv = 1 (the context owns the dense KV)", cfg->dense_tail_rows);
    }
    if (cfg->shared_spill != 0) {   // shared spill: requests that share a slot spill into it, each seeing only its own spilled keys
        MPIG_REQUIRE(cfg->shared_spill == 1, MPIG_EINVAL, "mpig_create: shared_spill = %d is not 0 or 1", cfg->shared_spill);
        MPIG_REQUIRE(cfg->num_contexts > 0 && cfg->num_contexts < cfg->batch_size && cfg->batch_size <= 32, MPIG_EINVAL,
                     "mpig_create: shared_spill needs fewer context slots than requests and at most 32 requests (one "
                     "visibility bit each): num_contexts = %d, batch_size = %d", cfg->num_contexts, cfg->batch_size);
    }
    for (int i = 0; i < 4; ++i)
        MPIG_REQUIRE(cfg->reserved[i] == 0, MPIG_EINVAL, "mpig_create: reserved[%d] = %d must be zero", i, cfg->reserved[i]);
    struct RestoreDevice {
        int prev = -1;
        RestoreDevice() { if (cudaGetDevice(&prev) != cudaSuccess) prev = -1; }
        ~RestoreDevice() { if (prev >= 0) cudaSetDevice(prev); }
    } restore_device;  // the caller's current device is left as it was found
    MPIG_CUDA(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    MPIG_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
    MPIG_REQUIRE(prop.major == 9 && prop.minor == 0, MPIG_EUNSUPPORTED,
                 "mpig_create: device %d is sm_%d%d; this library is built for sm_90a (H100) only and has no fallback",
                 cfg->device, prop.major, prop.minor);

    int ctx_max_cluster = 8;
    mpig_ctx *ctx = new mpig_ctx();
    ctx->cfg = *cfg;
    ctx->NB = 1 << cfg->K;
    // Key segments: at least ceil(M / 65536) (uint16 items), and as many as the CTAs a probing cluster will have -- then every CTA
    // of the cluster owns a WHOLE segment and streams only its own buckets (with fewer segments than CTAs, the CTAs sharing a
    // segment each stream all of its candidates and keep a sub-range: the same bucket bytes and sweep instructions r times over)
    {
        int c_target = 1;
        // `occ` CTAs of the probing / fused kernels share an SM (ctas_per_sm; default 1: one 1024-thread CTA per SM; 2: clusters
        // twice as large made of 512-thread CTAs, two per SM, whose latency phases overlap each other)
        const int occ = (cfg->ctas_per_sm == 2) ? 2 : 1;
        // ... and only while all B*Hq clusters stay resident at once: a cluster occupies SMs of ONE GPC and the H100's GPCs have
        // unequal SM counts, so fewer clusters of 4 fit than #SMs / 4 (a second wave of clusters doubles the launch)
        const long long heads = (long long)cfg->batch_size * cfg->num_attention_heads;
        while (c_target * 2 <= 8 && heads * c_target * 2 <= (long long)occ * prop.multiProcessorCount) {
            const int resident = fused_resident_clusters(c_target * 2, heads * c_target * 2 > prop.multiProcessorCount ? 512 : 1024);
            if (resident > 0 && heads > resident) break;
            c_target *= 2;
        }
        ctx_max_cluster = c_target;
        const int min_seg = (cfg->max_length + SEG - 1) / SEG;
        int nseg = std::max(min_seg, std::min(c_target, (cfg->max_length + 1023) / 1024));   // segments of < 1024 keys are not worth it
        int seg_len = (((cfg->max_length + nseg - 1) / nseg) + 63) & ~63;
        nseg = (cfg->max_length + seg_len - 1) / seg_len;   // rounding seg_len up may leave the last segment(s) empty
        ctx->nseg = std::max(nseg, 1);
        ctx->seg_len = seg_len;
    }
    ctx->Wcap = cfg->num_sink_tokens + cfg->num_local_tokens + cfg->generation_buffer;
    ctx->G = cfg->num_attention_heads / cfg->num_key_value_heads;
    ctx->H = cfg->batch_size * cfg->num_attention_heads;
    ctx->BG = cfg->batch_size * cfg->num_key_value_heads;
    ctx->rec_bytes = 2 * cfg->head_dim * 2;
    ctx->num_sms = prop.multiProcessorCount;
    ctx->cta_per_sm = (cfg->ctas_per_sm == 2) ? 2 : 1;
    ctx->max_cluster = ctx_max_cluster;
    ctx->bitmap_words = (cfg->max_length + 31) / 32;
    ctx->layers.resize(cfg->num_layers);
    ctx->C = cfg->num_contexts > 0 ? cfg->num_contexts : cfg->batch_size;
    ctx->n_off.assign(cfg->num_layers, std::vector<int>(ctx->C, 0));
    ctx->h_slot_of.resize(cfg->batch_size);
    for (int b = 0; b < cfg->batch_size; ++b) ctx->h_slot_of[b] = b % ctx->C;
    ctx->dense_tail_rows = cfg->dense_tail_rows;
    ctx->h_dense_base.assign(cfg->batch_size, 0);
    ctx->shared_spill = cfg->shared_spill == 1;
    ctx->h_private_lo.assign(cfg->num_layers, std::vector<int>(ctx->C, 0));

    const size_t M = (size_t)cfg->max_length, BG = (size_t)ctx->BG, L = (size_t)cfg->L, d = (size_t)cfg->head_dim;
    const size_t SG = (size_t)ctx->C * cfg->num_key_value_heads;   // slot groups: the store and the tables are per slot
    int rc = MPIG_OK;
#define TRY(x)                   \
    do {                         \
        rc = (x);                \
        if (rc != MPIG_OK) {     \
            mpig_destroy(ctx);   \
            return rc;           \
        }                        \
    } while (0)
    for (int l = 0; l < cfg->num_layers; ++l) {
        bool dense = false;
        for (int i = 0; i < cfg->num_dense_layers; ++i) dense |= (cfg->dense_layers[i] == l);
        LayerStore &ls = ctx->layers[l];
        if (dense) {
            ls.dense = true;
            if (cfg->alloc_dense_kv && ctx->dense_tail_rows > 0) {   // the slot stores and the request tails
                TRY(dev_alloc(ctx, &ls.dense_kv, SG * M * ctx->rec_bytes, false));
                TRY(dev_alloc(ctx, &ls.dense_tail, BG * (size_t)ctx->dense_tail_rows * ctx->rec_bytes, false));
            } else if (cfg->alloc_dense_kv) {
                TRY(dev_alloc(ctx, &ls.dense_kv, BG * M * ctx->rec_bytes, false));
            }
            continue;
        }
        ls.sparse = true;
        // zero-initialised like the reference's caches (sparse_attention.cc:563-581): an index >= n reads zeros, not garbage
        TRY(dev_alloc(ctx, &ls.kv, SG * M * ctx->rec_bytes, true));
        TRY(dev_alloc(ctx, &ls.kn, SG * M * sizeof(float), true));
        TRY(dev_alloc(ctx, &ls.offsets, SG * L * ctx->nseg * (size_t)(ctx->NB + 1) * sizeof(int32_t), true));
        TRY(dev_alloc(ctx, &ls.items, ((SG * L * M * sizeof(uint16_t) + 15) & ~(size_t)15), false));
        TRY(dev_alloc(ctx, &ls.win, BG * (size_t)(ctx->Wcap > 0 ? ctx->Wcap : 1) * ctx->rec_bytes, true));
        TRY(dev_alloc(ctx, &ls.avg_k, BG * d * sizeof(__nv_bfloat16), true));
    }
    const size_t H = (size_t)ctx->H;
    TRY(dev_alloc(ctx, &ctx->hash_func, d * cfg->K * L * sizeof(__nv_bfloat16)));
    TRY(dev_alloc(ctx, &ctx->hash_func_t, d * cfg->K * L * sizeof(__nv_bfloat16)));
    TRY(dev_alloc(ctx, &ctx->win_len, (size_t)cfg->batch_size * sizeof(int32_t)));
    TRY(dev_alloc(ctx, &ctx->dense_len, (size_t)cfg->batch_size * sizeof(int32_t)));
    TRY(dev_alloc(ctx, &ctx->slot_of, (size_t)cfg->batch_size * sizeof(int32_t)));
    if (ctx->dense_tail_rows > 0) TRY(dev_alloc(ctx, &ctx->dense_base, (size_t)cfg->batch_size * sizeof(int32_t)));
    if (ctx->shared_spill) {
        TRY(dev_alloc(ctx, &ctx->vis, (size_t)ctx->C * M * sizeof(uint32_t)));
        TRY(dev_alloc(ctx, &ctx->private_lo, (size_t)cfg->num_layers * ctx->C * sizeof(int32_t)));
    }
    // store_n [num_layers][C], allocated for C = batch_size so that a context's bytes per slot stay the store's and the tables'
    TRY(dev_alloc(ctx, &ctx->store_n, (size_t)cfg->num_layers * cfg->batch_size * sizeof(int32_t)));
    {
        const cudaError_t e = cudaMemcpy(ctx->slot_of, ctx->h_slot_of.data(), (size_t)cfg->batch_size * sizeof(int32_t),
                                         cudaMemcpyHostToDevice);
        if (e != cudaSuccess) {
            set_error("mpig_create: slot map upload failed: %s", cudaGetErrorString(e));
            mpig_destroy(ctx);
            return MPIG_ECUDA;
        }
    }
    TRY(dev_alloc(ctx, &ctx->codes, H * L * sizeof(int32_t)));
    TRY(dev_alloc(ctx, &ctx->qnorm, H * sizeof(float)));
    TRY(dev_alloc(ctx, &ctx->results, H * M * sizeof(int32_t)));
    TRY(dev_alloc(ctx, &ctx->nnz, H * sizeof(int32_t)));
    TRY(dev_alloc(ctx, &ctx->bitmaps, H * 2 * (size_t)ctx->bitmap_words * sizeof(uint32_t)));
    ctx->max_partial_warps = ctx->num_sms * 4 * 16;  // upper bound on warps of any attend launch
    TRY(dev_alloc(ctx, &ctx->partials, (size_t)ctx->max_partial_warps * 2 * 132 * sizeof(float)));
    TRY(dev_alloc(ctx, &ctx->counters, H * sizeof(int32_t)));
    TRY(dev_alloc(ctx, &ctx->mve, 2 * H * sizeof(float)));
    TRY(dev_alloc(ctx, &ctx->err_flag, 4 * sizeof(int32_t)));
    TRY(dev_alloc(ctx, &ctx->step_buf, (size_t)cfg->batch_size * (2 * TREE_MAX + 2) * sizeof(int32_t), true));
    TRY(dev_alloc(ctx, &ctx->slot_stage, (size_t)cfg->batch_size * sizeof(int32_t)));
    {   // layer table of mpig_accept and mpig_reorder_requests: every sparse window and every dense KV cache the context owns
        std::vector<AcceptLayer> tab;
        for (const LayerStore &ls : ctx->layers) {
            if (ls.sparse && ctx->Wcap > 0) tab.push_back({ls.win, ctx->Wcap, 0, ls.avg_k, 0});
            if (ls.dense && ls.dense_tail) tab.push_back({ls.dense_tail, ctx->dense_tail_rows, 1, nullptr, 0});
            else if (ls.dense && ls.dense_kv) tab.push_back({ls.dense_kv, cfg->max_length, 1, nullptr, 0});
        }
        int x0 = 0;
        for (AcceptLayer &e : tab) {
            e.x0 = x0;
            x0 += cfg->num_key_value_heads * ((e.cap + REORDER_ROWS - 1) / REORDER_ROWS);
        }
        ctx->reorder_cols = x0;
        ctx->n_accept_layers = (int)tab.size();
        if (!tab.empty()) {
            TRY(dev_alloc(ctx, (uint8_t **)&ctx->accept_layers, tab.size() * sizeof(AcceptLayer)));
            const cudaError_t e = cudaMemcpy(ctx->accept_layers, tab.data(), tab.size() * sizeof(AcceptLayer), cudaMemcpyHostToDevice);
            if (e != cudaSuccess) {
                set_error("mpig_create: accept table upload failed: %s", cudaGetErrorString(e));
                mpig_destroy(ctx);
                return MPIG_ECUDA;
            }
        }
    }
    ctx->h_win_len.assign(cfg->batch_size, 0);
    ctx->h_dense_len.assign(cfg->batch_size, 0);
    // staging of the *_host entry points: q | k | v | out, one MAPPED pinned block the kernels read and write directly
    const size_t stage = (((H * d + 2 * BG * d + H * d) * sizeof(__nv_bfloat16) + 255) & ~(size_t)255) + H * sizeof(uint32_t) + 256;
    TRY(dev_alloc(ctx, (uint8_t **)&ctx->dev_stage, stage));
    {
        cudaError_t e = cudaHostAlloc(&ctx->host_stage, stage, cudaHostAllocMapped);
        if (e == cudaSuccess) e = cudaHostGetDevicePointer(&ctx->host_stage_dev, ctx->host_stage, 0);
        if (e != cudaSuccess) {
            set_error("cudaHostAlloc(%zu, mapped) failed: %s", stage, cudaGetErrorString(e));
            mpig_destroy(ctx);
            return MPIG_ENOMEM;
        }
        memset(ctx->host_stage, 0, stage);
    }
#undef TRY
    MPIG_CUDA(cudaDeviceSynchronize());
    *out = ctx;
    return MPIG_OK;
}

}  // extern "C"

int mpig::upload_store_n(mpig_ctx *ctx, int layer, cudaStream_t s) {
    MPIG_CUDA(cudaMemcpyAsync(ctx->store_n + (size_t)layer * ctx->C, ctx->n_off[layer].data(), ctx->C * sizeof(int32_t),
                              cudaMemcpyHostToDevice, s));
    return MPIG_OK;
}

int mpig::refresh_maps(mpig_ctx *ctx, cudaStream_t s) {
    if (ctx->h_map_exact) return MPIG_OK;
    const int B = ctx->cfg.batch_size;
    std::vector<int32_t> so(B), db(B, 0);
    MPIG_CUDA(cudaMemcpyAsync(so.data(), ctx->slot_of, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (ctx->dense_base) MPIG_CUDA(cudaMemcpyAsync(db.data(), ctx->dense_base, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    MPIG_CUDA(cudaStreamSynchronize(s));
    for (int b = 0; b < B; ++b) {
        ctx->h_slot_of[b] = so[b];
        ctx->h_dense_base[b] = db[b];
    }
    return MPIG_OK;   // h_map_exact stays false: a later replay of the captured reorder changes the device maps again
}

extern "C" {

void mpig_destroy(mpig_ctx *ctx) {
    if (!ctx) return;
    {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    for (auto &ls : ctx->layers) {
        cudaFree(ls.kv);
        cudaFree(ls.kn);
        cudaFree(ls.offsets);
        cudaFree(ls.items);
        cudaFree(ls.win);
        cudaFree(ls.avg_k);
        cudaFree(ls.dense_kv);
        cudaFree(ls.dense_tail);
    }
    cudaFree(ctx->hash_func);
    cudaFree(ctx->hash_func_t);
    cudaFree(ctx->win_len);
    cudaFree(ctx->dense_len);
    cudaFree(ctx->slot_of);
    cudaFree(ctx->slot_stage);
    cudaFree(ctx->dense_base);
    cudaFree(ctx->vis);
    cudaFree(ctx->private_lo);
    cudaFree(ctx->store_n);
    cudaFree(ctx->chunk_partials);
    cudaFree(ctx->chunk_counters);
    cudaFree(ctx->codes);
    cudaFree(ctx->qnorm);
    cudaFree(ctx->results);
    cudaFree(ctx->nnz);
    cudaFree(ctx->bitmaps);
    cudaFree(ctx->partials);
    cudaFree(ctx->counters);
    cudaFree(ctx->mve);
    cudaFree(ctx->err_flag);
    cudaFree(ctx->step_buf);
    cudaFree(ctx->accept_layers);
    cudaFree(ctx->out_f32);
    cudaFree(ctx->dbg_buf);
    cudaFree(ctx->fused_dbg);
    free(ctx->fused_plan_cache);
    cudaFree(ctx->dev_stage);
    cudaFree(ctx->spill_buf);
    if (ctx->host_stage) cudaFreeHost(ctx->host_stage);
    for (auto e : ctx->timing_events) cudaEventDestroy(e);
    }
    delete ctx;
}

size_t mpig_device_bytes(const mpig_ctx *ctx) { return ctx ? ctx->bytes : 0; }
uint64_t mpig_launch_count(const mpig_ctx *ctx) { return ctx ? ctx->launches : 0; }

int mpig_clear(mpig_ctx *ctx, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "mpig_clear: null context");
    cudaStream_t s = as_stream(stream);
    const size_t BG = ctx->BG, SG = (size_t)ctx->C * ctx->cfg.num_key_value_heads, L = ctx->cfg.L;
    for (int l = 0; l < ctx->cfg.num_layers; ++l) {
        LayerStore &ls = ctx->layers[l];
        if (ls.sparse) {
            // an all-zero offsets array = every bucket empty; stale items/records are unreachable
            MPIG_CUDA(cudaMemsetAsync(ls.offsets, 0, SG * L * ctx->nseg * (size_t)(ctx->NB + 1) * sizeof(int32_t), s));
            MPIG_CUDA(cudaMemsetAsync(ls.avg_k, 0, BG * ctx->cfg.head_dim * sizeof(__nv_bfloat16), s));
        }
        for (auto &n : ctx->n_off[l]) n = 0;
    }
    MPIG_CUDA(cudaMemsetAsync(ctx->store_n, 0, (size_t)ctx->cfg.num_layers * ctx->C * sizeof(int32_t), s));
    MPIG_CUDA(cudaMemsetAsync(ctx->win_len, 0, ctx->cfg.batch_size * sizeof(int32_t), s));
    MPIG_CUDA(cudaMemsetAsync(ctx->dense_len, 0, ctx->cfg.batch_size * sizeof(int32_t), s));
    if (ctx->dense_base) MPIG_CUDA(cudaMemsetAsync(ctx->dense_base, 0, ctx->cfg.batch_size * sizeof(int32_t), s));
    for (auto &n : ctx->h_dense_base) n = 0;
    if (ctx->shared_spill) {   // no private keys: every slot's store is empty again
        MPIG_CUDA(cudaMemsetAsync(ctx->vis, 0, (size_t)ctx->C * ctx->cfg.max_length * sizeof(uint32_t), s));
        MPIG_CUDA(cudaMemsetAsync(ctx->private_lo, 0, (size_t)ctx->cfg.num_layers * ctx->C * sizeof(int32_t), s));
        for (auto &v : ctx->h_private_lo)
            for (auto &n : v) n = 0;
    }
    const size_t rows = (size_t)ctx->H * ctx->tok_max;   // the per-step scratch holds B*t_max*Hq rows after a reservation
    MPIG_CUDA(cudaMemsetAsync(ctx->nnz, 0, rows * sizeof(int32_t), s));
    MPIG_CUDA(cudaMemsetAsync(ctx->counters, 0, ctx->H * sizeof(int32_t), s));
    // lsh.cc:305 zeroes the mask: get_mask after clear must not return the previous probe's counters
    MPIG_CUDA(cudaMemsetAsync(ctx->bitmaps, 0, rows * 2 * ctx->bitmap_words * sizeof(uint32_t), s));
    MPIG_CUDA(cudaMemsetAsync(ctx->err_flag, 0, 4 * sizeof(int32_t), s));
    for (auto &n : ctx->h_win_len) n = 0;
    for (auto &n : ctx->h_dense_len) n = 0;
    // the initial binding b -> b mod C (the host mirror is a member: it outlives the copy)
    for (int b = 0; b < ctx->cfg.batch_size; ++b) ctx->h_slot_of[b] = b % ctx->C;
    MPIG_CUDA(cudaMemcpyAsync(ctx->slot_of, ctx->h_slot_of.data(), ctx->cfg.batch_size * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    ctx->h_len_exact = true;
    ctx->h_map_exact = !ctx->reorder_captured;
    ctx->last_tokens = 1;
    ctx->last_chunk = false;
    ctx->pending.end(true);   // no plan to decode, rewind or accept since the clear
    return MPIG_OK;
}

int mpig_set_hash_func(mpig_ctx *ctx, const void *hash_func_bf16, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx && hash_func_bf16, MPIG_EINVAL, "mpig_set_hash_func: null argument");
    cudaStream_t s = as_stream(stream);
    const int d = ctx->cfg.head_dim, KL = ctx->cfg.K * ctx->cfg.L;
    MPIG_CUDA(cudaMemcpyAsync(ctx->hash_func, hash_func_bf16, (size_t)d * KL * sizeof(__nv_bfloat16),
                              cudaMemcpyDefault, s));
    transpose_hash_func_kernel<<<(KL + 127) / 128, 128, 0, s>>>(ctx->hash_func, ctx->hash_func_t, d, KL);
    MPIG_LAUNCH_CHECK(ctx);
    ctx->hash_func_set = true;
    return MPIG_OK;
}

int mpig_set_option(mpig_ctx *ctx, const char *key, int64_t value) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx && key, MPIG_EINVAL, "mpig_set_option: null argument");
    std::string k(key);
    if (k == "save_mask") ctx->save_mask = (int)value;
    else if (k == "attend_ctas") ctx->attend.ctas = (int)value;
    else if (k == "attend_warps") ctx->attend.warps = (int)value;
    else if (k == "decode_impl") ctx->decode_impl = (int)value;
    else if (k == "fused_selcap") ctx->fused_selcap = value < 16 ? 16 : (value > 8192 ? 8192 : ((int)value + 15) & ~15);
    else if (k == "fused_kreg") ctx->fused_kreg = value ? 1 : 0;
    else if (k == "fused_issue_win") ctx->fused_issue_win = (int)std::max<int64_t>(0, std::min<int64_t>(value, 32));
    else if (k == "fused_debug") {
        ctx->fused_debug = (int)value;
        if (value && !ctx->fused_dbg) {
            MPIG_CUDA(cudaMalloc(&ctx->fused_dbg, (size_t)ctx->num_sms * 8 * 16 * sizeof(unsigned long long)));
            MPIG_CUDA(cudaMemset(ctx->fused_dbg, 0, (size_t)ctx->num_sms * 8 * 16 * sizeof(unsigned long long)));
        }
    }
    else if (k == "out_f32") {
        ctx->want_out_f32 = (int)value;
        if (value && !ctx->out_f32) {
            const size_t bytes = (size_t)ctx->H * std::max(ctx->tok_max, ctx->chunk_max) * ctx->cfg.head_dim * sizeof(float);
            MPIG_CUDA(cudaMalloc(&ctx->out_f32, bytes));
            MPIG_CUDA(cudaMemset(ctx->out_f32, 0, bytes));
        }
    }
    else if (k == "attend_tma") ctx->attend.tma = (int)value;
    else if (k == "dense_impl") ctx->dense_impl = (int)value;
    else if (k == "keyhash_impl") ctx->keyhash_impl = (int)value;
    else if (k == "pdl_first") ctx->pdl_first = (int)value;
    else if (k == "keyhash_skip") ctx->keyhash_skip = (int)value;
    else if (k == "attend_skip") ctx->attend_skip = (int)value;
    else if (k == "attend_debug") {
        ctx->attend_debug = (int)value;
        if (value && !ctx->dbg_buf) MPIG_CUDA(cudaMalloc(&ctx->dbg_buf, (size_t)ctx->max_partial_warps * 16 * sizeof(unsigned long long)));
    }
    else {
        set_error("mpig_set_option: unknown key '%s'", key);
        return MPIG_EINVAL;
    }
    return MPIG_OK;
}

int mpig_debug_read(mpig_ctx *ctx, unsigned long long *host_out, int nwarps) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx && host_out && ctx->dbg_buf, MPIG_EINVAL, "mpig_debug_read: debug not enabled");
    MPIG_REQUIRE(nwarps >= 0 && nwarps <= ctx->max_partial_warps, MPIG_EINVAL, "mpig_debug_read: nwarps=%d outside [0,%d]", nwarps,
                 ctx->max_partial_warps);
    MPIG_CUDA(cudaMemcpy(host_out, ctx->dbg_buf, (size_t)nwarps * 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return MPIG_OK;
}

int mpig_last_codes(mpig_ctx *ctx, int32_t *codes_out, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx && codes_out, MPIG_EINVAL, "mpig_last_codes: null argument");
    MPIG_REQUIRE(!ctx->last_chunk, MPIG_ESTATE, "mpig_last_codes: the last call was a chunk step (no LSH sample)");
    MPIG_REQUIRE(!ctx->last_decode_fused || ctx->save_mask, MPIG_ESTATE,
                 "mpig_last_codes: the fused decode keeps the query codes in shared memory; set option save_mask before the decode");
    MPIG_CUDA(cudaMemcpyAsync(codes_out, ctx->codes, (size_t)ctx->H * ctx->last_tokens * ctx->cfg.L * sizeof(int32_t),
                              cudaMemcpyDeviceToDevice, as_stream(stream)));
    return MPIG_OK;
}

int mpig_reserve_query_tokens(mpig_ctx *ctx, int t_max) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "mpig_reserve_query_tokens: null context");
    MPIG_REQUIRE(t_max >= 1 && t_max <= 8, MPIG_EINVAL, "mpig_reserve_query_tokens: t_max=%d outside [1, 8]", t_max);
    if (t_max <= ctx->tok_max) return MPIG_OK;
    // the scratch moves to new addresses: a step captured before would replay on freed memory
    MPIG_REQUIRE(!ctx->plan_captured, MPIG_ESTATE,
                 "mpig_reserve_query_tokens: a step has been captured into a CUDA graph; reserve before capturing");
    // the per-step scratch grows from B*Hq to B*t_max*Hq rows; the first B*Hq rows keep their meaning for single-token calls.
    // Everything is allocated first, so a failed allocation leaves the context as it was.
    const size_t H = (size_t)ctx->H * t_max, L = ctx->cfg.L, M = ctx->cfg.max_length, d = ctx->cfg.head_dim;
    const size_t sz[7] = {H * L * sizeof(int32_t), H * sizeof(float), H * M * sizeof(int32_t), H * sizeof(int32_t),
                          H * 2 * (size_t)ctx->bitmap_words * sizeof(uint32_t), 2 * H * sizeof(float),
                          (size_t)ctx->H * std::max(t_max, ctx->chunk_max) * d * sizeof(float)};   // out_f32 also serves chunk steps
    const int n = ctx->out_f32 ? 7 : 6;
    void *nb[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    MPIG_CUDA(cudaDeviceSynchronize());   // scratch of a decode still in flight is about to be freed
    for (int i = 0; i < n; ++i) {
        cudaError_t e = cudaMalloc(&nb[i], sz[i]);
        if (e == cudaSuccess) e = cudaMemset(nb[i], 0, sz[i]);
        if (e != cudaSuccess) {
            for (int j = 0; j <= i; ++j) cudaFree(nb[j]);
            (void)cudaGetLastError();
            set_error("mpig_reserve_query_tokens: cudaMalloc(%zu bytes) failed: %s", sz[i], cudaGetErrorString(e));
            return MPIG_ENOMEM;
        }
    }
    void **old[7] = {(void **)&ctx->codes, (void **)&ctx->qnorm, (void **)&ctx->results, (void **)&ctx->nnz, (void **)&ctx->bitmaps,
                     (void **)&ctx->mve, (void **)&ctx->out_f32};
    const size_t old_rows = (size_t)ctx->H * ctx->tok_max;
    for (int i = 0; i < n; ++i) {
        cudaFree(*old[i]);
        *old[i] = nb[i];
        if (i < 6) ctx->bytes += sz[i] - sz[i] / H * old_rows;   // (out_f32, an option's buffer, is not counted)
    }
    ctx->tok_max = t_max;
    return MPIG_OK;
}

int mpig_reserve_chunk_tokens(mpig_ctx *ctx, int t_max) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "mpig_reserve_chunk_tokens: null context");
    MPIG_REQUIRE(t_max >= 1 && t_max <= 1024, MPIG_EINVAL, "mpig_reserve_chunk_tokens: t_max=%d outside [1, 1024]", t_max);
    if (t_max <= ctx->chunk_max) return MPIG_OK;
    MPIG_REQUIRE(!ctx->plan_captured, MPIG_ESTATE,
                 "mpig_reserve_chunk_tokens: a step has been captured into a CUDA graph; reserve before capturing");
    // split states (a fixed size: see chunk_partial_tiles), merge tickets per m-block of t_max tokens, and the out_f32 copy grown to
    // B*t_max*Hq rows when the option has allocated it.  Everything is allocated first: a failed allocation changes nothing.
    const size_t sz[3] = {ctx->chunk_partials ? 0 : chunk_partial_bytes(ctx), (size_t)chunk_counter_count(ctx, t_max) * sizeof(int32_t),
                          ctx->out_f32 ? (size_t)ctx->H * std::max(t_max, ctx->tok_max) * ctx->cfg.head_dim * sizeof(float) : 0};
    void *nb[3] = {nullptr, nullptr, nullptr};
    MPIG_CUDA(cudaDeviceSynchronize());   // scratch of a step still in flight is about to be freed
    for (int i = 0; i < 3; ++i) {
        if (!sz[i]) continue;
        cudaError_t e = cudaMalloc(&nb[i], sz[i]);
        if (e == cudaSuccess) e = cudaMemset(nb[i], 0, sz[i]);
        if (e != cudaSuccess) {
            for (int j = 0; j <= i; ++j) cudaFree(nb[j]);
            (void)cudaGetLastError();
            set_error("mpig_reserve_chunk_tokens: cudaMalloc(%zu bytes) failed: %s", sz[i], cudaGetErrorString(e));
            return MPIG_ENOMEM;
        }
    }
    if (nb[0]) {
        ctx->chunk_partials = (float *)nb[0];
        ctx->chunk_part_tiles = chunk_partial_tiles(ctx);
        ctx->bytes += sz[0];
    }
    if (ctx->chunk_counters) ctx->bytes -= (size_t)chunk_counter_count(ctx, ctx->chunk_max) * sizeof(int32_t);
    cudaFree(ctx->chunk_counters);
    ctx->chunk_counters = (int32_t *)nb[1];
    ctx->bytes += sz[1];
    if (nb[2]) {
        cudaFree(ctx->out_f32);
        ctx->out_f32 = (float *)nb[2];
    }
    ctx->chunk_max = t_max;
    return MPIG_OK;
}

int mpig_fused_debug_read(mpig_ctx *ctx, unsigned long long *host_out, int nctas) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx && host_out && ctx->fused_dbg, MPIG_EINVAL, "mpig_fused_debug_read: option fused_debug not enabled");
    MPIG_REQUIRE(nctas >= 0 && nctas <= ctx->num_sms * 8, MPIG_EINVAL, "mpig_fused_debug_read: nctas=%d outside [0,%d]", nctas, ctx->num_sms * 8);
    MPIG_CUDA(cudaMemcpy(host_out, ctx->fused_dbg, (size_t)nctas * 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return MPIG_OK;
}

int mpig_error_flags(mpig_ctx *ctx, int32_t *flags_out, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx && flags_out, MPIG_EINVAL, "mpig_error_flags: null argument");
    int32_t f[4] = {0, 0, 0, 0};
    MPIG_CUDA(cudaMemcpyAsync(f, ctx->err_flag, sizeof(f), cudaMemcpyDeviceToHost, as_stream(stream)));
    MPIG_CUDA(cudaStreamSynchronize(as_stream(stream)));
    *flags_out = f[0];
    return MPIG_OK;
}

int mpig_last_out_f32(mpig_ctx *ctx, float *out_f32, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx && out_f32, MPIG_EINVAL, "mpig_last_out_f32: null argument");
    MPIG_REQUIRE(ctx->want_out_f32 && ctx->out_f32, MPIG_ESTATE, "mpig_last_out_f32: enable mpig_set_option(ctx, \"out_f32\", 1) before the decode");
    MPIG_CUDA(cudaMemcpyAsync(out_f32, ctx->out_f32, (size_t)ctx->H * ctx->last_tokens * ctx->cfg.head_dim * sizeof(float),
                              cudaMemcpyDeviceToDevice, as_stream(stream)));
    return MPIG_OK;
}

int mpig_get_info(mpig_ctx *ctx, const char *key, int64_t *value) {
    MPIG_REQUIRE(ctx && key && value, MPIG_EINVAL, "mpig_get_info: null argument");
    std::string k(key);
    if (k == "last_decode_fused") *value = ctx->last_decode_fused;
    else if (k == "fused_applicable") *value = fused_applicable(ctx) ? 1 : 0;
    else if (k == "fused_cluster_waves") *value = fused_cluster_waves(ctx);
    else if (k == "window_capacity") *value = ctx->Wcap;
    else if (k == "table_segments") *value = ctx->nseg;
    else if (k == "query_tokens_max") *value = ctx->tok_max;
    else if (k == "tokens_cluster_waves") *value = ctx->last_tokens_waves;
    else if (k == "num_contexts") *value = ctx->C;
    else if (k == "dense_tail_rows") *value = ctx->dense_tail_rows;
    else if (k == "shared_spill") *value = ctx->shared_spill ? 1 : 0;
    else if (k == "chunk_tokens_max") *value = ctx->chunk_max;
    else if (k == "chunk_splits") *value = ctx->last_chunk_splits;
    else {
        set_error("mpig_get_info: unknown key '%s'", key);
        return MPIG_EINVAL;
    }
    return MPIG_OK;
}

// shared checks of mpig_fork_request / mpig_bind_request
static int binding_checks(mpig_ctx *ctx, int request, const char *who) {
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "%s: null context", who);
    MPIG_REQUIRE(request >= 0 && request < ctx->cfg.batch_size, MPIG_EINVAL, "%s: request %d out of range [0, %d)", who, request,
                 ctx->cfg.batch_size);
    MPIG_REQUIRE(ctx->C < ctx->cfg.batch_size, MPIG_ESTATE,
                 "%s: every request owns its context slot (num_contexts = batch_size); create the context with fewer slots to share one",
                 who);
    return MPIG_OK;
}

static int upload_slot_map(mpig_ctx *ctx, cudaStream_t s) {
    MPIG_CUDA(cudaMemcpyAsync(ctx->slot_of, ctx->h_slot_of.data(), ctx->cfg.batch_size * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    MPIG_CUDA(cudaStreamSynchronize(s));
    return MPIG_OK;
}

int mpig_fork_request(mpig_ctx *ctx, int src, int dst, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    int rc = binding_checks(ctx, src, "mpig_fork_request");
    if (rc) return rc;
    rc = binding_checks(ctx, dst, "mpig_fork_request");
    if (rc) return rc;
    MPIG_REQUIRE(src != dst, MPIG_EINVAL, "mpig_fork_request: src == dst (%d)", src);
    cudaStream_t s = as_stream(stream);
    rc = refresh_maps(ctx, s);
    if (rc) return rc;
    int32_t len[2] = {0, 0};
    rc = read_lengths(ctx, src, 1, &len[0], &len[1], s);
    if (rc) return rc;
    const size_t Hkv = ctx->cfg.num_key_value_heads, REC = ctx->rec_bytes;
    for (const LayerStore &ls : ctx->layers) {
        if (ls.sparse) {
            const size_t pitch = (size_t)ctx->Wcap * REC;   // one kv-head's window
            if (len[0] > 0)
                MPIG_CUDA(cudaMemcpy2DAsync(ls.win + dst * Hkv * pitch, pitch, ls.win + src * Hkv * pitch, pitch, (size_t)len[0] * REC,
                                            Hkv, cudaMemcpyDeviceToDevice, s));
            const size_t avg = Hkv * ctx->cfg.head_dim;
            MPIG_CUDA(cudaMemcpyAsync(ls.avg_k + dst * avg, ls.avg_k + src * avg, avg * sizeof(__nv_bfloat16), cudaMemcpyDeviceToDevice, s));
        } else if (ls.dense_tail) {
            // shared dense mode: the prompt stays in the slot store; only src's tail rows [0, len - base) are copied
            const size_t pitch = (size_t)ctx->dense_tail_rows * REC;   // one kv-head's tail
            const int rows = std::min(std::max(len[1] - ctx->h_dense_base[src], 0), ctx->dense_tail_rows);
            if (rows > 0)
                MPIG_CUDA(cudaMemcpy2DAsync(ls.dense_tail + dst * Hkv * pitch, pitch, ls.dense_tail + src * Hkv * pitch, pitch,
                                            (size_t)rows * REC, Hkv, cudaMemcpyDeviceToDevice, s));
        } else if (ls.dense_kv && len[1] > 0) {
            const size_t pitch = (size_t)ctx->cfg.max_length * REC;   // one kv-head's cache
            MPIG_CUDA(cudaMemcpy2DAsync(ls.dense_kv + dst * Hkv * pitch, pitch, ls.dense_kv + src * Hkv * pitch, pitch,
                                        (size_t)len[1] * REC, Hkv, cudaMemcpyDeviceToDevice, s));
        }
    }
    if (ctx->dense_base) {
        MPIG_CUDA(cudaMemcpyAsync(ctx->dense_base + dst, ctx->dense_base + src, sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
        ctx->h_dense_base[dst] = ctx->h_dense_base[src];
    }
    MPIG_CUDA(cudaMemcpyAsync(ctx->win_len + dst, ctx->win_len + src, sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    MPIG_CUDA(cudaMemcpyAsync(ctx->dense_len + dst, ctx->dense_len + src, sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    ctx->h_win_len[dst] = len[0];
    ctx->h_dense_len[dst] = len[1];
    ctx->h_slot_of[dst] = ctx->h_slot_of[src];
    rc = launch_vis_rebind(ctx, src, dst, s);   // shared spill mode: dst sees exactly the private keys src sees
    if (rc) return rc;
    rc = upload_slot_map(ctx, s);
    if (rc) return rc;
    ctx->pending.end();   // its bases are stale for dst
    return MPIG_OK;
}

int mpig_bind_request(mpig_ctx *ctx, int request, int slot, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    int rc = binding_checks(ctx, request, "mpig_bind_request");
    if (rc) return rc;
    MPIG_REQUIRE(slot >= 0 && slot < ctx->C, MPIG_EINVAL, "mpig_bind_request: slot %d out of range [0, %d)", slot, ctx->C);
    rc = refresh_maps(ctx, as_stream(stream));   // the whole host map is uploaded below
    if (rc) return rc;
    ctx->h_slot_of[request] = slot;
    rc = launch_vis_rebind(ctx, -1, request, as_stream(stream));   // shared spill mode: no private key until it spills again
    if (rc) return rc;
    rc = upload_slot_map(ctx, as_stream(stream));
    if (rc) return rc;
    ctx->pending.end();
    return MPIG_OK;
}

int mpig_last_probe(mpig_ctx *ctx, int32_t *nnz_out, int32_t *results_out, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx && nnz_out, MPIG_EINVAL, "mpig_last_probe: null argument");
    MPIG_REQUIRE(!ctx->last_chunk, MPIG_ESTATE, "mpig_last_probe: the last call was a chunk step (no LSH sample)");
    const size_t rows = (size_t)ctx->H * ctx->last_tokens;
    MPIG_CUDA(cudaMemcpyAsync(nnz_out, ctx->nnz, rows * sizeof(int32_t), cudaMemcpyDeviceToDevice, as_stream(stream)));
    if (results_out)
        MPIG_CUDA(cudaMemcpyAsync(results_out, ctx->results, rows * ctx->cfg.max_length * sizeof(int32_t),
                                  cudaMemcpyDeviceToDevice, as_stream(stream)));
    return MPIG_OK;
}

}  // extern "C"
