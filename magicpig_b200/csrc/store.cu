// store.cu -- the HBM-resident KV store of the sparse layers and the operator entry points around stage 3.
//
// Replaces library/sparse_attention/sparse_attention.cc:
//   SparseAttentionServer::fill          :601-627   -> pack_records_kernel (K|V interleaved 512-byte records + fp32 norms)
//   get_key_cache / get_value_cache / get_key_norm :1213-1234 -> unpack_records_kernel
//   attention_wrapper                    :629-745   -> mpig_attention_wrapper (launches attend_mma_kernel, attend_mma.cu)
// and the dense layers' prefill copy (attnserver.py:116-120) -> pack_records_nhd_kernel; mpig_spill_window (no reference
// equivalent: generated window rows -> store + tables) -> spill_move_kernel, mpig_hash_keys, table_merge_kernel (tables.cu);
// mpig_compact_context (dead private keys out of a shared context) -> compact_live_kernel, compact_move_kernel,
// compact_stage_kernel, mpig_hash_keys, table_truncate_kernel and table_merge_kernel (tables.cu).
#include "attend_common.cuh"
#include "probe_common.cuh"

namespace mpig {

// ---------------------------------------------------------------------------------------------
// KV store maintenance
// ---------------------------------------------------------------------------------------------
// k, v (Hkv, n, D) bf16 -> records[(g*M + j)] = {k row | v row};  kn (Hkv, n) -> kn_store[g*M + j]
__global__ void pack_records_kernel(const uint4 *__restrict__ k, const uint4 *__restrict__ v, const float *__restrict__ kn,
                                    uint4 *__restrict__ rec, float *__restrict__ kn_store, int Hkv, int n, int rows_cap) {
    const size_t total = (size_t)Hkv * n * 32;  // 16-byte chunks per record: 16 K + 16 V
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int chunk = (int)(t & 31);
        const size_t row = t >> 5;  // g*n + j
        const int g = (int)(row / n), j = (int)(row % n);
        const uint4 val = (chunk < 16) ? k[row * 16 + chunk] : v[row * 16 + (chunk - 16)];
        rec[((size_t)g * rows_cap + j) * 32 + chunk] = val;
        if (chunk == 0 && kn) kn_store[(size_t)g * rows_cap + j] = kn[row];
    }
}

// records -> k, v (B, Hkv, M, D) / kn: the get_key_cache / get_value_cache / get_key_norm views
__global__ void unpack_records_kernel(const uint4 *__restrict__ rec, uint4 *__restrict__ k, uint4 *__restrict__ v,
                                      size_t rows) {
    const size_t total = rows * 32;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int chunk = (int)(t & 31);
        const size_t row = t >> 5;
        const uint4 val = rec[t];
        if (chunk < 16) {
            if (k) k[row * 16 + chunk] = val;
        } else {
            if (v) v[row * 16 + (chunk - 16)] = val;
        }
    }
}

// dense-layer fill: k, v (P, Hkv, D) NHD -> records[(g*M + j)]
__global__ void pack_records_nhd_kernel(const uint4 *__restrict__ k, const uint4 *__restrict__ v, uint4 *__restrict__ rec,
                                        int Hkv, int n, int rows_cap) {
    const size_t total = (size_t)Hkv * n * 32;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int chunk = (int)(t & 31);
        const size_t row = t >> 5;  // j*Hkv + g
        const int j = (int)(row / Hkv), g = (int)(row % Hkv);
        const uint4 val = (chunk < 16) ? k[row * 16 + chunk] : v[row * 16 + (chunk - 16)];
        rec[((size_t)g * rows_cap + j) * 32 + chunk] = val;
    }
}

// Window spill, store side (mpig_spill_window): one CTA per (kv-head, request) of one sparse layer, 8 warps.  The requests of a
// slot c spill into it one after the other: request b, bound to c = req_slot[b], owns rows off = req_off[b] .. off + g - 1 of
// the slot's g_c = slot_g[c] new rows.  With g = req_g[b]:
//   window rows [sink, sink + g) -> records n_old[c] + off .. + g - 1 of the slot's store (bitwise), their key norms
//   kn = bf16(||k||_2) widened to fp32 (fp32 sum of squares, one rounding: what fill() stores), and their key halves -> the
//   slot's staging block for the key hash, (Hkv, g_c, d) bf16 at row slot_pre[c] * Hkv, at offset off of every kv-head's run
//   (so the slot's new keys are hashed and merged together);
//   window rows [sink + g, sink + g + keep) -> [sink, sink + keep).
// With vis != null (shared spill mode, one sparse layer's launch: the map is the same for every layer) the CTAs of kv-head 0
// also make private keys slot_priv[c] + off .. + g - 1 of the slot visible to b alone.
// The kept rows move down in place, so they are copied in chunks of ascending rows, each chunk read completely before any of
// it is written (a row is only ever written after every row it lands on has been read).  One CTA owns the whole window of its
// (request, kv-head): no ordering between CTAs is involved.
__global__ void __launch_bounds__(256) spill_move_kernel(uint4 *win, uint4 *__restrict__ rec, float *__restrict__ kn_store,
                                                         uint4 *__restrict__ stage, const int32_t *__restrict__ req_g,
                                                         const int32_t *__restrict__ req_slot, const int32_t *__restrict__ req_off,
                                                         const int32_t *__restrict__ slot_g, const int32_t *__restrict__ slot_pre,
                                                         const int32_t *__restrict__ n_old, int Hkv, int M, int Wcap, int sink, int keep,
                                                         const int32_t *__restrict__ slot_priv, uint32_t *__restrict__ vis) {
    constexpr int T = 256, UN = 4;
    const int gi = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = req_g[b];
    if (g == 0) return;
    const int c = req_slot[b], off = req_off[b];
    const size_t bg = (size_t)b * Hkv + gi;
    const size_t sg = (size_t)c * Hkv + gi;   // store side: the request's slot
    uint4 *w = win + bg * Wcap * 32;
    uint4 *r = rec + (sg * M + n_old[c] + off) * 32;
    float *kns = kn_store + sg * M + n_old[c] + off;
    uint4 *st = stage + ((size_t)slot_pre[c] * Hkv + (size_t)gi * slot_g[c] + off) * 16;
    if (vis && gi == 0)
        for (int j = tid; j < g; j += T) vis[(size_t)c * M + slot_priv[c] + off + j] = 1u << b;
    for (int j = warp; j < g; j += T / 32) {
        const uint4 x = w[(size_t)(sink + j) * 32 + lane];
        r[(size_t)j * 32 + lane] = x;
        float ss = 0.f;
        if (lane < 16) {   // lanes 0..15 hold the key half of the record
            st[(size_t)j * 16 + lane] = x;
            const uint32_t p[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float a = bf16lo(p[i]), c = bf16hi(p[i]);
                ss = fmaf(a, a, ss);
                ss = fmaf(c, c, ss);
            }
        }
        ss = warp_sum(ss);
        if (lane == 0) kns[j] = __uint_as_float((uint32_t)f32_to_bf16_rne(sqrtf(ss)) << 16);
    }
    __syncthreads();
    const int total = keep * 32;   // 16-byte chunks of the kept rows
    uint4 *src = w + (size_t)(sink + g) * 32, *dst = w + (size_t)sink * 32;
    for (int c0 = 0; c0 < total; c0 += T * UN) {
        uint4 v[UN];
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const int i = c0 + u * T + tid;
            if (i < total) v[u] = src[i];
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const int i = c0 + u * T + tid;
            if (i < total) dst[i] = v[u];
        }
        __syncthreads();
    }
}

// shared spill mode, mpig_fork_request (src >= 0: dst sees exactly what src sees) and mpig_bind_request (src < 0: dst sees nothing)
__global__ void vis_rebind_kernel(uint32_t *vis, size_t words, int src, int dst) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t v = vis[i];
        vis[i] = (v & ~(1u << dst)) | (src >= 0 ? ((v >> src) & 1u) << dst : 0u);
    }
}

// shared spill mode, a fill: the slot's map is emptied and its private keys start at n in this layer
__global__ void reset_private_kernel(uint32_t *vis_slot, int M, int32_t *plo, int n) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < M; i += gridDim.x * blockDim.x) vis_slot[i] = 0u;
    if (blockIdx.x == 0 && threadIdx.x == 0) *plo = n;
}

int launch_vis_rebind(mpig_ctx *ctx, int src, int dst, cudaStream_t s) {
    if (!ctx->shared_spill) return MPIG_OK;
    const size_t words = (size_t)ctx->C * ctx->cfg.max_length;
    const int blocks = (int)std::min<size_t>((words + 255) / 256, (size_t)ctx->num_sms * 4);
    vis_rebind_kernel<<<blocks, 256, 0, s>>>(ctx->vis, words, src, dst);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

int reset_private(mpig_ctx *ctx, int layer, int request, int n, cudaStream_t s) {
    if (!ctx->shared_spill) return MPIG_OK;
    const int slot = ctx->h_slot_of[request], M = ctx->cfg.max_length;
    const int blocks = std::min((M + 255) / 256, ctx->num_sms * 4);
    reset_private_kernel<<<blocks, 256, 0, s>>>(ctx->vis + (size_t)slot * M, M, ctx->private_lo + (size_t)layer * ctx->C + slot, n);
    MPIG_LAUNCH_CHECK(ctx);
    ctx->h_private_lo[layer][slot] = n;
    return MPIG_OK;
}

// ---------------------------------------------------------------------------------------------
// Compaction (mpig_compact_context, shared spill mode): the slot's private keys that no request sees any more are dropped, the
// live ones keep their time order and move down to the offsets 0 .. live - 1.
// ---------------------------------------------------------------------------------------------
// Live list: one CTA per slot.  The ascending offsets p in [0, priv[c]) with vis[c][p] != 0 -> list[list_pre[c] ...], their
// count -> live[c].
__global__ void __launch_bounds__(1024) compact_live_kernel(const uint32_t *__restrict__ vis, int M, const int32_t *__restrict__ priv,
                                                            const int32_t *__restrict__ list_pre, int32_t *__restrict__ list,
                                                            int32_t *__restrict__ live) {
    __shared__ int wsum[40];
    const int c = blockIdx.x, n = priv[c];
    int32_t *out = list + list_pre[c];
    int base = 0;
    for (int p0 = 0; p0 < n; p0 += 1024) {
        const int p = p0 + (int)threadIdx.x;
        const int f = p < n && vis[(size_t)c * M + p] != 0u;
        int tot;
        const int ex = block_exclusive_scan(f, wsum, &tot);
        if (f) out[base + ex] = p;
        base += tot;
    }
    if (threadIdx.x == 0) live[c] = base;
}

struct CompactLayer {
    uint4 *kv;
    float *kn;
    const int32_t *plo;   // [C] the layer's private starts
};

// Record move, in place: one CTA per (kv-head, slot, sparse layer).  Live key j of a slot with work[c] moves from store index
// plo + list[j] to plo + j, record and key norm.  Sources ascend and every destination is at or below its source, so the rows
// are moved in ascending chunks, each chunk read completely before any of it is written: a write lands only on a row already
// read.  The CTA (0, c, 0) then moves the slot's vis words the same way and zeroes the words past the live count.
__global__ void __launch_bounds__(1024) compact_move_kernel(const CompactLayer *__restrict__ layers, const int32_t *__restrict__ list,
                                                            const int32_t *__restrict__ list_pre, const int32_t *__restrict__ live,
                                                            const int32_t *__restrict__ work, const int32_t *__restrict__ priv,
                                                            uint32_t *vis, int Hkv, int M) {
    constexpr int T = 1024, UN = 4, ROWS = T * UN / 32;   // 128 records (64 KB) per chunk
    const int gi = blockIdx.x, c = blockIdx.y, tid = threadIdx.x;
    if (!work[c]) return;
    const CompactLayer ly = layers[blockIdx.z];
    const int n = live[c], plo = ly.plo[c];
    const int32_t *src = list + list_pre[c];
    const size_t sg = (size_t)c * Hkv + gi;
    uint4 *r = ly.kv + (sg * M + plo) * 32;
    float *kns = ly.kn + sg * M + plo;
    for (int j0 = 0; j0 < n; j0 += ROWS) {
        uint4 v[UN];
        float kv_n = 0.f;
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const int j = j0 + u * (T / 32) + (tid >> 5);
            if (j < n) v[u] = r[(size_t)src[j] * 32 + (tid & 31)];
        }
        if (tid < ROWS && j0 + tid < n) kv_n = kns[src[j0 + tid]];
        __syncthreads();
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const int j = j0 + u * (T / 32) + (tid >> 5);
            if (j < n) r[(size_t)j * 32 + (tid & 31)] = v[u];
        }
        if (tid < ROWS && j0 + tid < n) kns[j0 + tid] = kv_n;
        __syncthreads();
    }
    if (gi != 0 || blockIdx.z != 0) return;
    uint32_t *vs = vis + (size_t)c * M;
    for (int j0 = 0; j0 < n; j0 += T) {
        const int j = j0 + tid;
        const uint32_t w = j < n ? vs[src[j]] : 0u;
        __syncthreads();
        if (j < n) vs[j] = w;
        __syncthreads();
    }
    for (int j = n + tid; j < priv[c]; j += T) vs[j] = 0u;
}

// The key halves of a slot's compacted live records [plo, plo + live) of one sparse layer -> its staging block for the key
// hash, (Hkv, live, d) bf16 at row spre[c] * Hkv, the layout the spill stages in.  grid (x, C).
__global__ void compact_stage_kernel(const uint4 *__restrict__ rec, const int32_t *__restrict__ plo, const int32_t *__restrict__ live,
                                     const int32_t *__restrict__ work, const int32_t *__restrict__ spre, uint4 *__restrict__ stage,
                                     int Hkv, int M) {
    const int c = blockIdx.y;
    if (!work[c]) return;
    const int n = live[c], p = plo[c];
    const size_t total = (size_t)Hkv * n * 16;
    uint4 *st = stage + (size_t)spre[c] * Hkv * 16;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const size_t row = t >> 4;   // gi * n + j
        const int gi = (int)(row / n), j = (int)(row % n);
        st[t] = rec[(((size_t)c * Hkv + gi) * M + p + j) * 32 + (t & 15)];
    }
}

// shared spill mode: private keys have the same offsets in every sparse layer only while the layers agree on a slot's private
// count.  priv[c] = that count for every slot with want[c] (0 for the others); MPIG_ESTATE when two sparse layers disagree.
static int private_counts(const mpig_ctx *ctx, const std::vector<char> &want, std::vector<int> &priv, const char *who) {
    const int C = ctx->C;
    priv.assign(C, -1);
    for (int l = 0; l < ctx->cfg.num_layers; ++l) {
        if (!ctx->layers[l].sparse) continue;
        for (int c = 0; c < C; ++c) {
            if (!want[c]) continue;
            const int pc = ctx->n_off[l][c] - ctx->h_private_lo[l][c];
            MPIG_REQUIRE(priv[c] < 0 || priv[c] == pc, MPIG_ESTATE,
                         "%s: context slot %d holds %d private keys in layer %d but %d in an earlier sparse layer "
                         "(a partial refill?); refill every sparse layer of the slot", who, c, pc, l, priv[c]);
            priv[c] = pc;
        }
    }
    for (int c = 0; c < C; ++c) priv[c] = std::max(priv[c], 0);
    return MPIG_OK;
}

int launch_pack_nhd(mpig_ctx *ctx, const void *k, const void *v, uint8_t *rec, int Hkv, int n, int rows_cap, cudaStream_t s) {
    const size_t total = (size_t)Hkv * n * 32;
    const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)ctx->num_sms * 16);
    pack_records_nhd_kernel<<<blocks, 256, 0, s>>>((const uint4 *)k, (const uint4 *)v, (uint4 *)rec, Hkv, n, rows_cap);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

}  // namespace mpig

using namespace mpig;

extern "C" {

int mpig_attn_fill(mpig_ctx *ctx, int layer, int request, const void *k_bf16, const void *v_bf16, const float *kn, int n,
                   void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_attn_fill");
    if (rc) return rc;
    MPIG_REQUIRE(request >= 0 && request < ctx->cfg.batch_size, MPIG_EINVAL, "mpig_attn_fill: request %d out of range", request);
    MPIG_REQUIRE(n >= 0 && n <= ctx->cfg.max_length, MPIG_EINVAL, "mpig_attn_fill: n=%d exceeds max_length=%d", n,
                 ctx->cfg.max_length);
    MPIG_REQUIRE(n == 0 || (k_bf16 && v_bf16 && kn), MPIG_EINVAL, "mpig_attn_fill: null input");
    const LayerStore &ls = ctx->layers[layer];
    const int Hkv = ctx->cfg.num_key_value_heads, M = ctx->cfg.max_length;
    rc = refresh_maps(ctx, as_stream(stream));
    if (rc) return rc;
    const int slot = ctx->h_slot_of[request];   // every request bound to this slot sees the new context
    rc = reset_private(ctx, layer, request, n, as_stream(stream));
    if (rc) return rc;
    ctx->n_off[layer][slot] = n;
    rc = upload_store_n(ctx, layer, as_stream(stream));
    if (rc) return rc;
    if (n == 0) return MPIG_OK;
    uint4 *rec = reinterpret_cast<uint4 *>(ls.kv + (size_t)slot * Hkv * M * ctx->rec_bytes);
    float *kns = ls.kn + (size_t)slot * Hkv * M;
    const size_t total = (size_t)Hkv * n * 32;
    const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)ctx->num_sms * 16);
    pack_records_kernel<<<blocks, 256, 0, as_stream(stream)>>>((const uint4 *)k_bf16, (const uint4 *)v_bf16, kn, rec, kns, Hkv,
                                                              n, M);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

int mpig_attention_wrapper(mpig_ctx *ctx, int layer, int K, int L, void *output_bf16, float *max_value_expsum, const void *query_bf16,
                           const float *query_norm, const int32_t *ind, const int32_t *nnz, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_attention_wrapper");
    if (rc) return rc;
    MPIG_REQUIRE(output_bf16 && max_value_expsum && query_bf16 && query_norm && ind && nnz, MPIG_EINVAL,
                 "mpig_attention_wrapper: null argument");
    MPIG_REQUIRE(K >= 1 && K <= 15 && L >= 1 && L <= 1024, MPIG_EINVAL, "mpig_attention_wrapper: K=%d L=%d outside [1,15] x [1,1024]", K, L);
    const LayerStore &ls = ctx->layers[layer];
    AttendParams p = attend_params(ctx, query_bf16, query_norm, output_bf16);
    p.kv = ls.kv;
    p.kn = ls.kn;
    p.slot_of = ctx->slot_map();
    p.ind = ind;
    p.nnz = nnz;
    p.mve = max_value_expsum;
    p.K = K;
    p.L = L;
    ctx->last_tokens = 1;
    ctx->last_chunk = false;
    return launch_attend_mma(ctx, p, as_stream(stream), false);
}

int mpig_attn_read_cache(mpig_ctx *ctx, int layer, void *k_bf16, void *v_bf16, float *kn, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_attn_read_cache");
    if (rc) return rc;
    const LayerStore &ls = ctx->layers[layer];
    const size_t rows = (size_t)ctx->C * ctx->cfg.num_key_value_heads * ctx->cfg.max_length;   // every slot
    if (k_bf16 || v_bf16) {
        const int blocks = (int)std::min<size_t>((rows * 32 + 255) / 256, (size_t)ctx->num_sms * 16);
        unpack_records_kernel<<<blocks, 256, 0, as_stream(stream)>>>((const uint4 *)ls.kv, (uint4 *)k_bf16, (uint4 *)v_bf16,
                                                                    rows);
        MPIG_LAUNCH_CHECK(ctx);
    }
    if (kn) MPIG_CUDA(cudaMemcpyAsync(kn, ls.kn, rows * sizeof(float), cudaMemcpyDeviceToDevice, as_stream(stream)));
    return MPIG_OK;
}

int mpig_spill_window(mpig_ctx *ctx, int keep, int32_t *spilled_out, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "mpig_spill_window: null context");
    const int B = ctx->cfg.batch_size, sink = ctx->cfg.num_sink_tokens, M = ctx->cfg.max_length;
    const int Hkv = ctx->cfg.num_key_value_heads, L = ctx->cfg.L, d = ctx->cfg.head_dim, nl = ctx->cfg.num_layers;
    MPIG_REQUIRE(keep >= 0 && sink + keep < ctx->Wcap, MPIG_EINVAL,
                 "mpig_spill_window: keep=%d: sink (%d) + keep must leave a free row in the window (capacity %d)", keep, sink, ctx->Wcap);
    MPIG_REQUIRE(ctx->hash_func_set, MPIG_ESTATE, "mpig_spill_window before mpig_set_hash_func: the spilled keys cannot be hashed");
    cudaStream_t s = as_stream(stream);
    std::vector<int32_t> wl(B);
    int rc = read_lengths(ctx, 0, B, wl.data(), nullptr, s);
    if (rc) return rc;
    rc = refresh_maps(ctx, s);   // each request's keys go to the slot it is bound to now
    if (rc) return rc;
    // The spill is planned per context slot: the requests of a slot spill into its store in request order, and the slot's new
    // keys are staged as one block, the blocks in slot order, so that they are hashed and merged together.
    // meta = per request g[B] | slot[B] | off[B] (the rows the slot's earlier requests spill) | per slot g[C] (the sum over its
    // requests) | pre[C] (its staging block) | priv[C] (its first new private offset, shared spill mode) | n_old[num_layers][C]
    const int C = ctx->C;
    const size_t o_slot = B, o_off = 2 * (size_t)B, o_sg = 3 * (size_t)B, o_spre = o_sg + C, o_priv = o_spre + C, o_n = o_priv + C;
    std::vector<int32_t> meta(o_n + (size_t)nl * C, 0);
    const std::vector<int> &slot = ctx->h_slot_of;
    for (int b = 0; b < B; ++b) {
        const int g = std::max(0, wl[b] - sink - keep);
        meta[b] = g;
        meta[o_slot + b] = slot[b];
        meta[o_off + b] = meta[o_sg + slot[b]];
        meta[o_sg + slot[b]] += g;
    }
    int tot = 0;
    for (int c = 0; c < C; ++c) {
        meta[o_spre + c] = tot;
        tot += meta[o_sg + c];
    }
    if (ctx->shared_spill) {
        std::vector<char> want(C);
        for (int c = 0; c < C; ++c) want[c] = meta[o_sg + c] > 0;
        std::vector<int> priv;
        rc = private_counts(ctx, want, priv, "mpig_spill_window");
        if (rc) return rc;
        for (int c = 0; c < C; ++c) meta[o_priv + c] = priv[c];
    } else {
        // a shared slot's store and tables are every bound request's context: spilling one request's generated tokens into them
        // would put those tokens into the others' samples
        for (int b = 0; b < B; ++b)
            for (int o = 0; o < B && meta[b] > 0; ++o)
                MPIG_REQUIRE(o == b || slot[o] != slot[b] || wl[o] == 0, MPIG_ESTATE,
                             "mpig_spill_window: request %d would spill %d rows into context slot %d, which request %d (window of %d rows) "
                             "shares; a shared request generates at most generation_buffer tokens unless the context was created "
                             "with shared spill (mpig_config.shared_spill)", b, meta[b], slot[b], o, wl[o]);
    }
    for (int l = 0; l < nl; ++l) {
        if (!ctx->layers[l].sparse) continue;
        for (int c = 0; c < C; ++c) {
            const int n_old = ctx->n_off[l][c];
            MPIG_REQUIRE(n_old + meta[o_sg + c] <= M, MPIG_ESTATE,
                         "mpig_spill_window: layer %d context slot %d: %d offloaded + %d spilled keys exceed max_length=%d", l, c,
                         n_old, meta[o_sg + c], M);
            meta[o_n + (size_t)l * C + c] = n_old;
        }
    }
    if (tot > 0) {
        // scratch for the worst case (every request spills all its non-sink rows), allocated once
        const size_t meta_bytes = ((meta.size() * sizeof(int32_t)) + 255) & ~(size_t)255;
        const size_t rows_cap = (size_t)B * std::max(ctx->Wcap - sink, 1);
        const size_t key_bytes = rows_cap * Hkv * d * sizeof(__nv_bfloat16);
        if (!ctx->spill_buf) {
            const size_t bytes = meta_bytes + key_bytes + rows_cap * Hkv * L * sizeof(int16_t);
            cudaError_t e = cudaMalloc(&ctx->spill_buf, bytes);
            if (e != cudaSuccess) {
                ctx->spill_buf = nullptr;
                (void)cudaGetLastError();
                set_error("mpig_spill_window: cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
                return MPIG_ENOMEM;
            }
            ctx->bytes += bytes;
        }
        int32_t *d_meta = reinterpret_cast<int32_t *>(ctx->spill_buf);
        __nv_bfloat16 *keys = reinterpret_cast<__nv_bfloat16 *>(ctx->spill_buf + meta_bytes);
        int16_t *codes = reinterpret_cast<int16_t *>(ctx->spill_buf + meta_bytes + key_bytes);
        MPIG_CUDA(cudaMemcpyAsync(d_meta, meta.data(), meta.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        bool vis_done = false;
        for (int l = 0; l < nl; ++l) {
            LayerStore &ls = ctx->layers[l];
            if (!ls.sparse) continue;
            const int32_t *n_old = d_meta + o_n + (size_t)l * C;
            spill_move_kernel<<<dim3(Hkv, B), 256, 0, s>>>(reinterpret_cast<uint4 *>(ls.win), reinterpret_cast<uint4 *>(ls.kv), ls.kn,
                                                          reinterpret_cast<uint4 *>(keys), d_meta, d_meta + o_slot, d_meta + o_off,
                                                          d_meta + o_sg, d_meta + o_spre, n_old, Hkv, M, ctx->Wcap, sink, keep,
                                                          d_meta + o_priv, ctx->shared_spill && !vis_done ? ctx->vis : nullptr);
            MPIG_LAUNCH_CHECK(ctx);
            vis_done = true;
            for (int c = 0; c < C; ++c) {
                const int g = meta[o_sg + c], pre = meta[o_spre + c];
                if (g == 0) continue;
                const int rc = mpig_hash_keys(ctx, keys + (size_t)pre * Hkv * d, g, codes + (size_t)pre * Hkv * L, stream);
                if (rc) return rc;
            }
            const int rc = launch_table_merge(ctx, l, codes, d_meta + o_sg, d_meta + o_spre, n_old, s);
            if (rc) return rc;
        }
        for (int b = 0; b < B; ++b)
            if (meta[b] > 0) wl[b] = sink + keep;
        MPIG_CUDA(cudaMemcpyAsync(ctx->win_len, wl.data(), B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        // the pageable host buffers above must outlive the copies
        MPIG_CUDA(cudaStreamSynchronize(s));
        for (int l = 0; l < nl; ++l)
            if (ctx->layers[l].sparse) {
                for (int c = 0; c < C; ++c) ctx->n_off[l][c] += meta[o_sg + c];
                rc = upload_store_n(ctx, l, s);
                if (rc) return rc;
            }
        if (ctx->h_len_exact)
            for (int b = 0; b < B; ++b) ctx->h_win_len[b] = wl[b];
    }
    if (spilled_out)
        for (int b = 0; b < B; ++b) spilled_out[b] = meta[b];
    return MPIG_OK;
}

int mpig_read_visibility(mpig_ctx *ctx, uint32_t *vis_out, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx && vis_out, MPIG_EINVAL, "mpig_read_visibility: null argument");
    MPIG_REQUIRE(ctx->shared_spill, MPIG_ESTATE, "mpig_read_visibility: the context has no shared spill (mpig_config.shared_spill)");
    MPIG_CUDA(cudaMemcpyAsync(vis_out, ctx->vis, (size_t)ctx->C * ctx->cfg.max_length * sizeof(uint32_t), cudaMemcpyDeviceToDevice,
                              as_stream(stream)));
    return MPIG_OK;
}

// scratch of one compaction, freed on every return
struct CompactScratch {
    std::vector<void *> bufs;
    ~CompactScratch() {
        for (void *p : bufs) (void)cudaFree(p);
    }
    int alloc(size_t bytes, void **p) {
        cudaError_t e = cudaMalloc(p, std::max<size_t>(bytes, 16));
        if (e != cudaSuccess) {
            (void)cudaGetLastError();
            set_error("mpig_compact_context: cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
            return MPIG_ENOMEM;
        }
        bufs.push_back(*p);
        return MPIG_OK;
    }
};

int mpig_compact_context(mpig_ctx *ctx, int slot, int32_t *reclaimed_out, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "mpig_compact_context: null context");
    const int C = ctx->C, M = ctx->cfg.max_length, nl = ctx->cfg.num_layers;
    const int Hkv = ctx->cfg.num_key_value_heads, L = ctx->cfg.L, d = ctx->cfg.head_dim;
    MPIG_REQUIRE(slot >= -1 && slot < C, MPIG_EINVAL, "mpig_compact_context: slot %d outside [-1, %d)", slot, C);
    if (reclaimed_out)
        for (int c = 0; c < C; ++c) reclaimed_out[c] = 0;
    if (!ctx->shared_spill) return MPIG_OK;   // no private keys
    MPIG_REQUIRE(ctx->hash_func_set, MPIG_ESTATE, "mpig_compact_context before mpig_set_hash_func: the live keys cannot be rehashed");
    cudaStream_t s = as_stream(stream);
    std::vector<char> want(C, 0);
    for (int c = 0; c < C; ++c) want[c] = slot < 0 || c == slot;
    std::vector<int> priv;
    int rc = private_counts(ctx, want, priv, "mpig_compact_context");
    if (rc) return rc;
    std::vector<int> sparse;
    for (int l = 0; l < nl; ++l)
        if (ctx->layers[l].sparse) sparse.push_back(l);
    const int nsl = (int)sparse.size();
    // meta = list_pre[C] | priv[C] | live[C] | work[C] | spre[C] | g[C] (live where work, else 0: the keys merged back) |
    // lo[nsl][C] | hi[nsl][C], then the layer table
    const size_t o_priv = C, o_live = 2 * (size_t)C, o_work = 3 * (size_t)C, o_spre = 4 * (size_t)C, o_g = 5 * (size_t)C,
                 o_lo = 6 * (size_t)C, o_hi = o_lo + (size_t)nsl * C;
    std::vector<int32_t> meta(o_hi + (size_t)nsl * C, 0);
    int tot_priv = 0;
    for (int c = 0; c < C; ++c) {
        meta[c] = tot_priv;
        meta[o_priv + c] = priv[c];
        tot_priv += priv[c];
    }
    if (tot_priv == 0) return MPIG_OK;
    const size_t meta_bytes = (meta.size() * sizeof(int32_t) + 255) & ~(size_t)255;
    const size_t table_bytes = (nsl * sizeof(CompactLayer) + 255) & ~(size_t)255;
    CompactScratch scratch;
    uint8_t *small = nullptr;
    rc = scratch.alloc(meta_bytes + table_bytes + (size_t)tot_priv * sizeof(int32_t), (void **)&small);
    if (rc) return rc;
    int32_t *d_meta = reinterpret_cast<int32_t *>(small);
    CompactLayer *d_layers = reinterpret_cast<CompactLayer *>(small + meta_bytes);
    int32_t *d_list = reinterpret_cast<int32_t *>(small + meta_bytes + table_bytes);
    // 1. the live lists and counts (nothing is written to the context before the scratch below is allocated)
    MPIG_CUDA(cudaMemcpyAsync(d_meta, meta.data(), 2 * C * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    compact_live_kernel<<<C, 1024, 0, s>>>(ctx->vis, M, d_meta + o_priv, d_meta, d_list, d_meta + o_live);
    MPIG_LAUNCH_CHECK(ctx);
    MPIG_CUDA(cudaMemcpyAsync(meta.data() + o_live, d_meta + o_live, C * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    MPIG_CUDA(cudaStreamSynchronize(s));
    int tot_live = 0, nwork = 0;
    for (int c = 0; c < C; ++c) {
        const int live = meta[o_live + c];
        meta[o_work + c] = want[c] && live < priv[c];
        meta[o_spre + c] = tot_live;
        if (!meta[o_work + c]) continue;
        ++nwork;
        meta[o_g + c] = live;
        tot_live += live;
    }
    if (nwork == 0) return MPIG_OK;
    std::vector<CompactLayer> table(nsl);
    for (int i = 0; i < nsl; ++i) {
        const int l = sparse[i];
        LayerStore &ls = ctx->layers[l];
        table[i] = {reinterpret_cast<uint4 *>(ls.kv), ls.kn, ctx->private_lo + (size_t)l * C};
        for (int c = 0; c < C; ++c) {
            const int lo = ctx->h_private_lo[l][c];
            meta[o_lo + (size_t)i * C + c] = lo;
            meta[o_hi + (size_t)i * C + c] = meta[o_work + c] ? ctx->n_off[l][c] : lo;   // lo == hi: the truncate leaves c alone
        }
    }
    // 2. hash scratch sized to the live keys of one layer: their key halves (Hkv, live, d) bf16 and codes (Hkv, L, live) int16
    const size_t key_bytes = ((size_t)tot_live * Hkv * d * sizeof(__nv_bfloat16) + 255) & ~(size_t)255;
    uint8_t *big = nullptr;
    rc = scratch.alloc(key_bytes + (size_t)tot_live * Hkv * L * sizeof(int16_t), (void **)&big);
    if (rc) return rc;
    __nv_bfloat16 *keys = reinterpret_cast<__nv_bfloat16 *>(big);
    int16_t *codes = reinterpret_cast<int16_t *>(big + key_bytes);
    MPIG_CUDA(cudaMemcpyAsync(d_meta, meta.data(), meta.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    MPIG_CUDA(cudaMemcpyAsync(d_layers, table.data(), nsl * sizeof(CompactLayer), cudaMemcpyHostToDevice, s));
    // 3. records, norms and the visibility map, every sparse layer in one launch
    compact_move_kernel<<<dim3(Hkv, C, nsl), 1024, 0, s>>>(d_layers, d_list, d_meta, d_meta + o_live, d_meta + o_work, d_meta + o_priv,
                                                           ctx->vis, Hkv, M);
    MPIG_LAUNCH_CHECK(ctx);
    // 4. per sparse layer: stage and hash the live keys, drop every private item from the tables, merge the live keys back
    for (int i = 0; i < nsl; ++i) {
        const int l = sparse[i];
        const int32_t *lo = d_meta + o_lo + (size_t)i * C;
        if (tot_live > 0) {
            const int blocks = (int)std::min<size_t>(((size_t)tot_live * Hkv * 16 + 255) / 256, (size_t)ctx->num_sms * 4);
            compact_stage_kernel<<<dim3(std::max(blocks / nwork, 1), C), 256, 0, s>>>(reinterpret_cast<const uint4 *>(ctx->layers[l].kv),
                                                                                    lo, d_meta + o_live, d_meta + o_work,
                                                                                    d_meta + o_spre, reinterpret_cast<uint4 *>(keys), Hkv, M);
            MPIG_LAUNCH_CHECK(ctx);
            for (int c = 0; c < C; ++c) {
                const int g = meta[o_live + c], pre = meta[o_spre + c];
                if (!meta[o_work + c] || g == 0) continue;
                rc = mpig_hash_keys(ctx, keys + (size_t)pre * Hkv * d, g, codes + (size_t)pre * Hkv * L, stream);
                if (rc) return rc;
            }
        }
        rc = launch_table_truncate(ctx, l, lo, d_meta + o_hi + (size_t)i * C, s);
        if (rc) return rc;
        rc = launch_table_merge(ctx, l, codes, d_meta + o_g, d_meta + o_spre, lo, s);
        if (rc) return rc;
    }
    MPIG_CUDA(cudaStreamSynchronize(s));
    for (int l : sparse) {
        for (int c = 0; c < C; ++c)
            if (meta[o_work + c]) ctx->n_off[l][c] = ctx->h_private_lo[l][c] + meta[o_live + c];
        rc = upload_store_n(ctx, l, s);
        if (rc) return rc;
    }
    MPIG_CUDA(cudaStreamSynchronize(s));
    if (reclaimed_out)
        for (int c = 0; c < C; ++c) reclaimed_out[c] = meta[o_work + c] ? priv[c] - meta[o_live + c] : 0;
    return MPIG_OK;
}

}  // extern "C"
