// attend_chunk.cu -- chunk steps (mpig_plan_chunk / mpig_chunk_attend): exact causal softmax attention of T <= 1024 new tokens per
// request over everything the request sees, on sparse and dense layers alike.  No sampling and no importance weights: this is the
// attention a prefill of the whole conversation computes, so a follow-up turn or a forked request's question can be fed in one
// pass per layer instead of T single-token steps.
//
// A CTA owns one (request b, kv-head h, m-block of 128 query rows, key split).  The T*G query rows of the kv-group are ordered
// r = t*G + g (token t, q-head h*G + g), so the causal limit of a row depends on t only.  The key axis of the request is two record
// ranges laid end to end:
//   range A (slot level)    sparse: the slot's sampled store [0, n_slot); in shared spill mode the private keys [plo, n_slot) the
//                           request does not see (vis bit b clear) are masked.  Dense with dense_tail_rows: the slot's prompt rows
//                           [0, dense_base[b]).  Default dense layout: empty.
//   range B (request level) sparse: the window; dense: the request's rows (or its tail); the step's T rows are its last T, so
//                           token t sees rows [0, base + t] of it.
// Every key of range A is visible to every row (up to the private filter), so with combined index k (A first) a key is visible to
// token t iff k <= nA + base + t: one comparison per score.  The combined axis is cut into `splits` equal ranges of whole 64-key
// tiles; the split states (m, l, o) of a tile's rows are merged by the last CTA to finish (merge_states, as attend_dense_kernel's
// level-2 merge), or finalised in registers when splits = 1.  The m-blocks of one (group, split) are adjacent in blockIdx.x, so they
// stream the same records through L2 at about the same time.
//
// Tensor cores: mma.sync m16n8k16 (bf16 in, fp32 accumulate), the fragment code of attend_dense_kernel: 8 warps x 16 query rows,
// Q fragments in registers for the whole key loop, K (ldmatrix) and V (ldmatrix.trans) from a ring of 64-record tiles that one warp
// fills with per-record cp.async.bulk copies into 528-byte slots (conflict-free ldmatrix without a swizzle).  P goes into P.V as
// bf16 hi + lo (the split of attend_dense_kernel): P rounded to plain bf16 misses 1e-3 of fp64 once a few keys take most of the
// probability (tests/test_chunk_cpu.py emulates both; DESIGN.md section 3.14).
#include "attend_common.cuh"

namespace mpig {

constexpr int CK_WARPS = 8;
constexpr int CK_ROWS = 16 * CK_WARPS;   // query rows per m-block
constexpr int CK_KT = 64;                // keys per tile
constexpr int CK_ST = 3;                 // tiles in flight (ring depth)
constexpr int CK_SPLIT_MAX = 16;
constexpr size_t CK_SMEM = (size_t)CK_ST * CK_KT * SLOT + CK_ST * sizeof(uint64_t);

struct ChunkParams {
    const uint8_t *a_rows;       // range A records [C*Hkv][M] (sparse store / dense slot store), null = no range A
    const int32_t *a_n;          // sparse: keys in the store per slot [C] (this layer)
    const int32_t *plo;          // shared spill: first private key per slot [C] (this layer), else null
    const uint32_t *vis;         // shared spill: [C][M] visibility bits of the private keys
    const int32_t *slot_of;      // [B] or null (request b reads slot b)
    const int32_t *dense_base;   // dense with tails: [B] first row of each request in its tail, else null
    const uint8_t *b_rows;       // range B records [B*Hkv][bcap]
    const int32_t *bases;        // step_bases(step_buf): [B][2] window / dense length before the step
    const __nv_bfloat16 *q;      // [B][T][Hq][D]
    __nv_bfloat16 *out;          // [B][T][Hq][D]
    float *out_f32;              // same or null
    float *partials;             // [tiles][splits][CK_ROWS][PART_FLOATS]
    int32_t *counters;           // [B*Hkv*nmb] merge tickets (self-resetting)
    int T, G, Hkv, Hq, M, bcap, dense, nmb, splits;
};

__device__ __forceinline__ void chunk_store_row(const ChunkParams &p, size_t o, int col, float v0, float v1, float inv) {
    const float a = v0 * inv, c = v1 * inv;
    if (p.out_f32) *reinterpret_cast<float2 *>(p.out_f32 + o * D + col) = make_float2(a, c);
    *reinterpret_cast<uint32_t *>(p.out + o * D + col) = (uint32_t)f32_to_bf16_half_up(a) | ((uint32_t)f32_to_bf16_half_up(c) << 16);
}

__global__ void __launch_bounds__(CK_WARPS * 32, 1) attend_chunk_kernel(const __grid_constant__ ChunkParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + (size_t)CK_ST * CK_KT * SLOT);
    __shared__ int s_ticket;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, grp = lane >> 2, tig = lane & 3;
    const int mb = blockIdx.x % p.nmb, sp = blockIdx.x / p.nmb, h = blockIdx.y, b = blockIdx.z;
    const int G = p.G, TG = p.T * G;
    if (threadIdx.x == 0) {
        for (int i = 0; i < CK_ST; ++i) mbar_init(&bar[i], 1);
        fence_mbar_init();
    }
    pdl_wait();   // the step's rows (append_tokens_kernel), the lengths, maps and q are written by earlier kernels
    const int slot = p.slot_of ? __ldg(p.slot_of + b) : b;
    int nA = 0, jb0, plo = 0x7fffffff;
    const uint8_t *A = nullptr;
    if (!p.dense) {
        nA = min(max(p.a_n[slot], 0), p.M);
        A = p.a_rows + ((size_t)slot * p.Hkv + h) * p.M * REC;
        if (p.plo) plo = p.plo[slot];
        jb0 = p.bases[2 * b];
    } else if (p.dense_base) {
        const int base = p.dense_base[b], step = p.bases[2 * b + 1];
        nA = min(max(min(base, step), 0), p.M);
        A = p.a_rows + ((size_t)slot * p.Hkv + h) * p.M * REC;
        jb0 = max(step - base, 0);
    } else {
        jb0 = p.bases[2 * b + 1];
    }
    jb0 = max(jb0, 0);
    const uint8_t *Bp = p.b_rows + ((size_t)b * p.Hkv + h) * p.bcap * REC;
    const int nB = min(jb0 + p.T, p.bcap);
    const int ntot = nA + nB;
    const int r0 = mb * CK_ROWS, rows_valid = min(CK_ROWS, TG - r0);
    const int t_hi = (r0 + rows_valid - 1) / G;
    const int kend_block = min(ntot, nA + jb0 + t_hi + 1);
    const int per = ((ntot + p.splits - 1) / p.splits + CK_KT - 1) / CK_KT * CK_KT;
    const int k_begin = sp * per, k_end = min(k_begin + per, kend_block);
    const int ntiles = (k_end > k_begin) ? (k_end - k_begin + CK_KT - 1) / CK_KT : 0;
    __syncthreads();   // barriers initialised
    pdl_launch_dependents();

    // warp 0 fills ring stage it % CK_ST with tile it: one bulk copy per record; slots past the range get a copy of the tile's first
    // record (finite values under a zero probability)
    auto rec = [&](int k) { return k < nA ? A + (size_t)k * REC : Bp + (size_t)(k - nA) * REC; };
    auto issue = [&](int it) {
        const int st = it % CK_ST, k0 = k_begin + it * CK_KT, cnt = min(CK_KT, k_end - k0);
        uint8_t *dst = smem + (size_t)st * CK_KT * SLOT;
        if (lane == 0) mbar_arrive_expect_tx(&bar[st], (uint32_t)CK_KT * REC);
        __syncwarp();
        for (int r = lane; r < CK_KT; r += 32) bulk_g2s(dst + (size_t)r * SLOT, rec(k0 + (r < cnt ? r : 0)), REC, &bar[st]);
    };
    if (warp == 0)
        for (int it = 0; it < min(CK_ST, ntiles); ++it) issue(it);

    // this lane's query rows r = r0 + warp*16 + i*8 + grp; lim = the last combined key index the row sees (-1: no row)
    const int wrow0 = r0 + warp * 16;
    const bool warp_live = wrow0 < TG;
    const uint32_t *qrow[2];
    int lim[2];
    size_t orow[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int r = wrow0 + i * 8 + grp;
        const bool ok = r < TG;
        const int t = ok ? r / G : 0, g = ok ? r % G : 0;
        orow[i] = ((size_t)b * p.T + t) * p.Hq + (size_t)h * G + g;
        qrow[i] = ok ? reinterpret_cast<const uint32_t *>(p.q + orow[i] * D) : nullptr;
        lim[i] = ok ? nA + jb0 + t : -1;
    }
    // every score of a tile below lim_lo (and below k_end, outside the private range) is visible to all 16 rows of the warp
    const int lim_lo = (wrow0 + 16 <= TG) ? nA + jb0 + wrow0 / G : -1;
    const int priv_lo = min(plo, nA);   // private keys: [priv_lo, nA) when plo < nA
    const uint32_t *vis_slot = p.vis ? p.vis + (size_t)slot * p.M : nullptr;

    uint32_t qa[8][4];
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
        qa[ks][0] = qrow[0] ? __ldg(qrow[0] + ks * 8 + tig) : 0u;
        qa[ks][1] = qrow[1] ? __ldg(qrow[1] + ks * 8 + tig) : 0u;
        qa[ks][2] = qrow[0] ? __ldg(qrow[0] + ks * 8 + 4 + tig) : 0u;
        qa[ks][3] = qrow[1] ? __ldg(qrow[1] + ks * 8 + 4 + tig) : 0u;
    }
    const float scale_log2 = rsqrtf((float)D) * LOG2E_F;
    const uint32_t k_lane_off = (uint32_t)(((lane & 7) + (lane >> 4) * 8) * SLOT + ((lane >> 3) & 1) * 16);
    const uint32_t v_lane_off = (uint32_t)(((lane & 7) + ((lane >> 3) & 1) * 8) * SLOT + D * 2 + (lane >> 4) * 16);
    float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_run[2] = {0.f, 0.f};
    float acc[16][4];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;

    for (int it = 0; it < ntiles; ++it) {
        const int st = it % CK_ST, k0 = k_begin + it * CK_KT;
        const uint32_t tile_s = smem_u32(smem + (size_t)st * CK_KT * SLOT);
        mbar_wait(&bar[st], (uint32_t)((it / CK_ST) & 1));
        if (warp_live) {
            // ---- S = Q . K^T: 16 rows x 64 keys per warp ------------------------------------------------------------------
            float s[8][4];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 8; ++ks)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    uint32_t kb[4];
                    ldsm_x4(kb, tile_s + (uint32_t)(j * 16 * SLOT + ks * 32) + k_lane_off);
                    mma_16816(s[2 * j], qa[ks], kb[0], kb[1]);
                    mma_16816(s[2 * j + 1], qa[ks], kb[2], kb[3]);
                }
            // ---- masks: causal limit, split end, private keys the request does not see -------------------------------------
            const bool priv_tile = priv_lo < nA && k0 + CK_KT > priv_lo && k0 < nA;
            const bool full = !priv_tile && k0 + CK_KT <= k_end && k0 + CK_KT - 1 <= lim_lo;
            uint32_t pmask = 0xffffu;   // bit nt*2 + e: this lane's key nt*8 + tig*2 + e passes the private filter
            if (priv_tile) {
#pragma unroll
                for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int k = k0 + nt * 8 + tig * 2 + e;
                        if (k >= priv_lo && k < nA && !((__ldg(vis_slot + (k - plo)) >> b) & 1u)) pmask &= ~(1u << (nt * 2 + e));
                    }
            }
            float corr[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float mloc = -CUDART_INF_F;
#pragma unroll
                for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float &x = s[nt][2 * i + e];
                        const int k = k0 + nt * 8 + tig * 2 + e;
                        const bool vis = full || (k < k_end && k <= lim[i] && ((pmask >> (nt * 2 + e)) & 1u));
                        x = vis ? x * scale_log2 : -CUDART_INF_F;
                        mloc = fmaxf(mloc, x);
                    }
                mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 1));
                mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 2));
                const float m_new = fmaxf(m_run[i], mloc);
                const float m_use = (m_new == -CUDART_INF_F) ? 0.f : m_new;   // a row with no visible key yet: all p = 0
                corr[i] = (m_run[i] == -CUDART_INF_F) ? 0.f : exp2f(m_run[i] - m_new);
                float lsum = 0.f;
#pragma unroll
                for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float &x = s[nt][2 * i + e];
                        x = exp2f(x - m_use);
                        lsum += x;
                    }
                lsum += __shfl_xor_sync(0xffffffffu, lsum, 1);
                lsum += __shfl_xor_sync(0xffffffffu, lsum, 2);
                l_run[i] = l_run[i] * corr[i] + lsum;
                m_run[i] = m_new;
            }
#pragma unroll
            for (int n = 0; n < 16; ++n) {
                acc[n][0] *= corr[0]; acc[n][1] *= corr[0];
                acc[n][2] *= corr[1]; acc[n][3] *= corr[1];
            }
            // ---- O += P . V, P as bf16 hi + lo -----------------------------------------------------------------------------
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                uint32_t ahi[4], alo[4];
#pragma unroll
                for (int half = 0; half < 2; ++half)
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const float p0 = s[2 * ks + half][2 * i], p1 = s[2 * ks + half][2 * i + 1];
                        const uint32_t h0 = f32_to_bf16_rne(p0), h1 = f32_to_bf16_rne(p1);
                        const uint32_t l0 = f32_to_bf16_rne(p0 - bf16_bits_to_f32(h0)), l1 = f32_to_bf16_rne(p1 - bf16_bits_to_f32(h1));
                        ahi[2 * half + i] = h0 | (h1 << 16);
                        alo[2 * half + i] = l0 | (l1 << 16);
                    }
#pragma unroll
                for (int n2 = 0; n2 < 8; ++n2) {
                    uint32_t vb[4];
                    ldsm_x4_trans(vb, tile_s + (uint32_t)(ks * 16 * SLOT + n2 * 32) + v_lane_off);
                    mma_16816(acc[2 * n2], ahi, vb[0], vb[1]);
                    mma_16816(acc[2 * n2 + 1], ahi, vb[2], vb[3]);
                    mma_16816(acc[2 * n2], alo, vb[0], vb[1]);
                    mma_16816(acc[2 * n2 + 1], alo, vb[2], vb[3]);
                }
            }
        }
        fence_proxy_async();   // this stage's generic reads before the async copies that refill it
        __syncthreads();
        if (warp == 0 && it + CK_ST < ntiles) issue(it + CK_ST);
    }

    if (p.splits == 1) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (!qrow[i]) continue;
            const float inv = (l_run[i] > 0.f) ? 1.0f / l_run[i] : 0.f;
#pragma unroll
            for (int n = 0; n < 16; ++n) chunk_store_row(p, orow[i], n * 8 + tig * 2, acc[n][2 * i], acc[n][2 * i + 1], inv);
        }
        return;
    }
    // ---- several splits: this split's states, then the last CTA of the tile merges them ---------------------------------------
    const size_t tile_id = ((size_t)b * p.Hkv + h) * p.nmb + mb;
    float *part = p.partials + (tile_id * p.splits + sp) * (size_t)CK_ROWS * PART_FLOATS;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (!qrow[i]) continue;
        float *stt = part + (size_t)(warp * 16 + i * 8 + grp) * PART_FLOATS;
        if (tig == 0) {
            stt[0] = m_run[i] * 0.6931471805599453f;   // natural-log units, as merge_states reads them
            stt[1] = l_run[i];
        }
#pragma unroll
        for (int n = 0; n < 16; ++n) *reinterpret_cast<float2 *>(stt + 4 + n * 8 + tig * 2) = make_float2(acc[n][2 * i], acc[n][2 * i + 1]);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_ticket = atom_add_acq_rel_gpu(p.counters + tile_id, 1);
    __syncthreads();
    if (s_ticket != p.splits - 1) return;
    for (int rr = warp; rr < rows_valid; rr += CK_WARPS) {
        float M_, L_, Acc[4];
        merge_states<true>([&](int i) { return (const float *)(p.partials + ((tile_id * p.splits + i) * CK_ROWS + rr) * (size_t)PART_FLOATS); },
                           p.splits, lane, M_, L_, Acc);
        const int r = r0 + rr, t = r / G, g = r % G;
        const size_t o = ((size_t)b * p.T + t) * p.Hq + (size_t)h * G + g;
        const float inv = (L_ > 0.f) ? 1.0f / L_ : 0.f;
        chunk_store_row(p, o, 4 * lane, Acc[0], Acc[1], inv);
        chunk_store_row(p, o, 4 * lane + 2, Acc[2], Acc[3], inv);
    }
    if (threadIdx.x == 0) p.counters[tile_id] = 0;
}

// append the T rows of layer `layer` (centred on a sparse layer, raw on a dense one), then the chunk attention under PDL
int launch_chunk_attend(mpig_ctx *ctx, int layer, int T, const void *q, const void *k, const void *v, void *out, cudaStream_t s) {
    const LayerStore &ls = ctx->layers[layer];
    const bool dense = ls.dense;
    const int B = ctx->cfg.batch_size, Hkv = ctx->cfg.num_key_value_heads;
    int rc = launch_append_tokens(ctx, append_params(ctx, ls, k, v, dense), T, s, dense ? ctx->dense_base_map() : nullptr);
    if (rc) return rc;
    ChunkParams p = {};
    const bool tail = dense && ctx->dense_tail_rows > 0;
    if (!dense) {
        p.a_rows = ls.kv;
        p.a_n = ctx->store_n + (size_t)layer * ctx->C;
        p.plo = ctx->private_lo_map(layer);
        p.vis = ctx->vis_map();
        p.b_rows = ls.win;
        p.bcap = ctx->Wcap;
    } else if (tail) {
        p.a_rows = ls.dense_kv;
        p.dense_base = ctx->dense_base;
        p.b_rows = ls.dense_tail;
        p.bcap = ctx->dense_tail_rows;
    } else {
        p.b_rows = ls.dense_kv;
        p.bcap = ctx->cfg.max_length;
    }
    p.slot_of = ctx->slot_map();
    p.bases = step_bases(ctx->step_buf, B);
    p.q = (const __nv_bfloat16 *)q;
    p.out = (__nv_bfloat16 *)out;
    p.out_f32 = ctx->want_out_f32 ? ctx->out_f32 : nullptr;
    p.partials = ctx->chunk_partials;
    p.counters = ctx->chunk_counters;
    p.T = T;
    p.G = ctx->G;
    p.Hkv = Hkv;
    p.Hq = ctx->cfg.num_attention_heads;
    p.M = ctx->cfg.max_length;
    p.dense = dense ? 1 : 0;
    p.nmb = (T * ctx->G + CK_ROWS - 1) / CK_ROWS;
    // key splits: enough CTAs for about two per SM when the m-blocks alone are fewer than the SMs, each split at least 512 keys of
    // the longest request (host mirrors; after a captured plan they are estimates, which changes the speed, never the result)
    const int ctas = p.nmb * Hkv * B;
    int keys = 0;
    for (int b = 0; b < B; ++b) {
        int n = dense ? ctx->h_dense_len[b] : ctx->n_off[layer][ctx->h_slot_of[b]] + ctx->h_win_len[b];
        if (!ctx->h_len_exact) n = dense ? ctx->cfg.max_length : ctx->cfg.max_length + ctx->Wcap;
        keys = std::max(keys, n);
    }
    int splits = (ctas < ctx->num_sms) ? std::min(CK_SPLIT_MAX, std::max(1, 2 * ctx->num_sms / ctas)) : 1;
    splits = std::max(1, std::min(splits, keys / 512));
    p.splits = splits;
    MPIG_REQUIRE(splits == 1 || (size_t)splits * ctas <= (size_t)ctx->chunk_part_tiles, MPIG_EINVAL,
                 "chunk attention: partial scratch too small (%d splits x %d tiles)", splits, ctas);
    MPIG_FUNC_ATTR(attend_chunk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CK_SMEM);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(p.nmb * splits, Hkv, B);
    cfg.blockDim = dim3(CK_WARPS * 32);
    cfg.dynamicSmemBytes = CK_SMEM;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    MPIG_CUDA(cudaLaunchKernelEx(&cfg, attend_chunk_kernel, p));
    MPIG_LAUNCH_CHECK(ctx);
    ctx->last_tokens = T;
    ctx->last_chunk = true;
    ctx->last_chunk_splits = splits;
    return MPIG_OK;
}

// the tiles the partial scratch of mpig_reserve_chunk_tokens holds: splits > 1 only while the m-blocks are fewer than the SMs, and
// then splits * m-blocks <= 2 * SMs
int chunk_partial_tiles(const mpig_ctx *ctx) { return 2 * ctx->num_sms; }
size_t chunk_partial_bytes(const mpig_ctx *ctx) { return (size_t)chunk_partial_tiles(ctx) * CK_ROWS * PART_FLOATS * sizeof(float); }
int chunk_counter_count(const mpig_ctx *ctx, int t_max) {
    return ctx->BG * ((t_max * ctx->G + CK_ROWS - 1) / CK_ROWS);
}

}  // namespace mpig
