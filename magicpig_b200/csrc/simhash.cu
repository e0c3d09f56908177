// simhash.cu -- SimHash of the decode queries, plus the row appends and the window fill.  The step lifecycle (plan, rewind,
// accept) is in step.cu.
//
// Replaces the GPU-side torch glue of LSHSparseAttnServer.decode:
//   attnserver.py:264-270   norm_q = q/||q|| (bf16) ; P = norm_q @ hash_func ; bit = P > 0 ;
//                           code[h,l] = sum_i bit[h, l*K+i] << i                 -> simhash_kernel
//   attnserver.py:300       ||q||_2 in fp32 of the bf16 query                     -> same kernel
//   attnserver.py:275-290   k_new -= avg_k ; append k_new, v_new to the window    -> same launch (extra CTA), or
//                                                                                    append_tokens_kernel
//   attnserver.py:142-153   window fill at prefill                                -> window_fill_kernel
//
// The projection is a (B*Hq x 128) x (128 x K*L) bf16 GEMM with fp32 accumulation on the tensor
// cores (mma.sync m16n8k16 -- 12 MFLOP per layer, launch-latency bound; one CTA per 8 tables so the
// 384 KB of hash_func is read exactly once per launch across the grid).  Only the SIGN of each
// accumulator leaves the register file: bits are packed little-endian per table (column l*K+i is
// bit i of table l) into int32 codes.
#include <algorithm>

#include "common.cuh"

namespace mpig {

constexpr int SH_D = 128;
constexpr int SH_STRIDE = SH_D + 8;   // bf16 elements; 272 B rows -> conflict-free fragment loads
constexpr int SH_TABLES = 8;          // tables per CTA -> 8*K columns = K n-tiles of 8
constexpr int SH_MBLOCK = 32;         // query rows per CTA (grid.y walks the row blocks)
constexpr int SH_THREADS = 256;


// One warp stores input row `row` of k_new / v_new as record `pos` of kv-group bg: 256 B of K (centred on avg_k when it is set,
// bf16 arithmetic as torch: fp32 subtract, RNE) + 256 B of V.
__device__ __forceinline__ void store_row(const AppendParams &a, int bg, int pos, int row, int lane) {
    uint8_t *rec = a.rows + ((size_t)bg * a.cap + pos) * (4 * SH_D);
    const size_t src = (size_t)row * SH_D + 4 * lane;
    const uint2 kk = *reinterpret_cast<const uint2 *>(a.k_new + src);
    uint2 ko = kk;
    if (a.avg_k) {
        const uint2 av = *reinterpret_cast<const uint2 *>(a.avg_k + (size_t)bg * SH_D + 4 * lane);
        ko.x = (uint32_t)f32_to_bf16_rne(bf16lo(kk.x) - bf16lo(av.x)) | ((uint32_t)f32_to_bf16_rne(bf16hi(kk.x) - bf16hi(av.x)) << 16);
        ko.y = (uint32_t)f32_to_bf16_rne(bf16lo(kk.y) - bf16lo(av.y)) | ((uint32_t)f32_to_bf16_rne(bf16hi(kk.y) - bf16hi(av.y)) << 16);
    }
    *reinterpret_cast<uint2 *>(rec + 8 * lane) = ko;
    *reinterpret_cast<uint2 *>(rec + 2 * SH_D + 8 * lane) = *reinterpret_cast<const uint2 *>(a.v_new + src);
}

// the new row of every (request, kv-head), (B, Hkv, D) -> position len[b] - 1: the warps of the CTA take the groups in turn
__device__ __forceinline__ void append_rows(const AppendParams &a) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
    for (int bg = warp; bg < a.BG; bg += warps) {
        const int b = bg / a.Hkv;
        const int pos = a.len[b] - 1;
        if (pos < 0 || pos >= a.cap) continue;
        store_row(a, bg, pos, bg, lane);
    }
}

__device__ __forceinline__ void mma_bf16_16816(float c[4], const uint32_t a[4], const uint32_t b[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// grid = (ceil(L / SH_TABLES) (+1 CTA for the append when a.k_new != null), ceil(H / SH_MBLOCK)), SH_THREADS threads
// dynamic smem: Qraw [SH_MBLOCK][128] bf16 | A [SH_MBLOCK][SH_STRIDE] bf16 | B [SH_TABLES*K][SH_STRIDE] bf16
//               | bits [SH_MBLOCK][SH_TABLES*K] u8
// Latency is the whole cost here, so every global load of a pass (the CTA's hash_func slice and the raw
// query rows) is issued up front as one batch of cp.async (LDGSTS) and waited on once.
__global__ void __launch_bounds__(SH_THREADS) simhash_kernel(const __nv_bfloat16 *__restrict__ q,        // (H, D)
                                                             const __nv_bfloat16 *__restrict__ hf_t,     // (K*L, D)
                                                             int32_t *__restrict__ codes,                // (H, L)
                                                             float *__restrict__ qnorm,                  // (H) or null
                                                             int H, int K, int L, int n_hash_ctas, AppendParams ap) {
    extern __shared__ __align__(16) uint8_t sh_smem[];
    const int ncols_max = SH_TABLES * K;
    __nv_bfloat16 *sQ = reinterpret_cast<__nv_bfloat16 *>(sh_smem);
    __nv_bfloat16 *sA = sQ + SH_MBLOCK * SH_D;
    __nv_bfloat16 *sB = sA + SH_MBLOCK * SH_STRIDE;
    uint8_t *sBits = reinterpret_cast<uint8_t *>(sB + ncols_max * SH_STRIDE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int NW = SH_THREADS / 32;
    const bool hash_cta = (int)blockIdx.x < n_hash_ctas;
    const int t0 = blockIdx.x * SH_TABLES;
    const int ntab = hash_cta ? min(SH_TABLES, L - t0) : 0;
    const int ncols = ntab * K;
    const int col0 = t0 * K;
    const int ncols_pad = (ncols + 7) & ~7;

    if (hash_cta) {
        // hash_func is constant data: its slice can be fetched before the producer kernel has finished
        for (int t = threadIdx.x; t < ncols_pad * 16; t += SH_THREADS) {
            const int c = t >> 4, ch = t & 15;
            uint8_t *dst = reinterpret_cast<uint8_t *>(sB + (size_t)c * SH_STRIDE) + ch * 16;
            if (c < ncols) cp_async16(dst, reinterpret_cast<const uint4 *>(hf_t + (size_t)(col0 + c) * SH_D) + ch);
            else *reinterpret_cast<uint4 *>(dst) = make_uint4(0, 0, 0, 0);
        }
    }
    pdl_launch_dependents();  // the probe may start its prologue; it still waits for this grid to finish
    pdl_wait();  // q / k_new / v_new come from the caller's previous kernel
    if (!hash_cta) {
        if (blockIdx.y == 0) append_rows(ap);
        return;
    }

    {
        const int m0 = blockIdx.y * SH_MBLOCK;   // this CTA's block of query rows
        const int mrows = min(SH_MBLOCK, H - m0);
        const int mrows_pad = (mrows + 15) & ~15;
        for (int t = threadIdx.x; t < mrows * 16; t += SH_THREADS)
            cp_async16(reinterpret_cast<uint8_t *>(sQ) + (size_t)t * 16, reinterpret_cast<const uint4 *>(q + (size_t)m0 * SH_D) + t);
        cp_async_wait_all();
        __syncthreads();
        // A block: norm_q rows, bf16 arithmetic exactly as torch does it (attnserver.py:265-266)
        for (int r = warp; r < mrows_pad; r += NW) {
            uint2 o = make_uint2(0, 0);
            if (r < mrows) {
                const uint2 v = *(reinterpret_cast<const uint2 *>(sQ + (size_t)r * SH_D) + lane);
                const float x0 = bf16lo(v.x), x1 = bf16hi(v.x), x2 = bf16lo(v.y), x3 = bf16hi(v.y);
                const float ss = warp_sum(x0 * x0 + x1 * x1 + x2 * x2 + x3 * x3);
                const float nrm32 = sqrtf(ss);
                if (qnorm && blockIdx.x == 0 && lane == 0) qnorm[m0 + r] = nrm32;  // fp32 norm (attnserver.py:300)
                const float nrm = bf16_bits_to_f32(f32_to_bf16_rne(nrm32));        // bf16-rounded norm
                o.x = (uint32_t)f32_to_bf16_rne(x0 / nrm) | ((uint32_t)f32_to_bf16_rne(x1 / nrm) << 16);
                o.y = (uint32_t)f32_to_bf16_rne(x2 / nrm) | ((uint32_t)f32_to_bf16_rne(x3 / nrm) << 16);
            }
            *reinterpret_cast<uint2 *>(reinterpret_cast<uint8_t *>(sA + (size_t)r * SH_STRIDE) + lane * 8) = o;
        }
        __syncthreads();
        // tensor-core projection: (m-tile, n-tile) pairs round-robin over the warps
        const int grp = lane >> 2, tig = lane & 3;
        const int n_mt = mrows_pad / 16, n_nt = ncols_pad / 8;
        for (int pair = warp; pair < n_mt * n_nt; pair += NW) {
            const int mt = pair / n_nt, nt = pair % n_nt;
            float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                const __nv_bfloat16 *base = sA + (size_t)(mt * 16 + grp) * SH_STRIDE + kk * 16 + tig * 2;
                uint32_t afr[4], bfr[2];
                afr[0] = *reinterpret_cast<const uint32_t *>(base);
                afr[1] = *reinterpret_cast<const uint32_t *>(base + 8 * SH_STRIDE);
                afr[2] = *reinterpret_cast<const uint32_t *>(base + 8);
                afr[3] = *reinterpret_cast<const uint32_t *>(base + 8 * SH_STRIDE + 8);
                const __nv_bfloat16 *bb = sB + (size_t)(nt * 8 + grp) * SH_STRIDE + kk * 16 + tig * 2;
                bfr[0] = *reinterpret_cast<const uint32_t *>(bb);
                bfr[1] = *reinterpret_cast<const uint32_t *>(bb + 8);
                mma_bf16_16816(c, afr, bfr);
            }
            // only the sign survives (attnserver.py:267 .gt(0))
            const int r0 = mt * 16 + grp, cc = nt * 8 + tig * 2;
            sBits[(size_t)r0 * ncols_max + cc] = c[0] > 0.f;
            sBits[(size_t)r0 * ncols_max + cc + 1] = c[1] > 0.f;
            sBits[(size_t)(r0 + 8) * ncols_max + cc] = c[2] > 0.f;
            sBits[(size_t)(r0 + 8) * ncols_max + cc + 1] = c[3] > 0.f;
        }
        __syncthreads();
        // little-endian pack per table (attnserver.py:268-270)
        for (int t = threadIdx.x; t < mrows * ntab; t += SH_THREADS) {
            const int r = t / ntab, tb = t % ntab;
            const uint8_t *bp = sBits + (size_t)r * ncols_max + tb * K;
            int code = 0;
            for (int i = 0; i < K; ++i) code |= (int)bp[i] << i;
            codes[(size_t)(m0 + r) * L + t0 + tb] = code;
        }
    }
}

// T new rows per (request, kv-head): one warp per (b, t, kv-head).  k_new / v_new are (B, T, Hkv, D); row t of request b goes to
// position len[b] - T + t (len already advanced by the plan); with a base map (shared dense mode: a.rows are the request tails)
// to position len[b] - T + t - base[b] of the tail.  The attention launch that reads the rows follows under programmatic
// dependent launch.
__global__ void append_tokens_kernel(AppendParams a, int T, const int32_t *base) {
    pdl_launch_dependents();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= a.BG * T) return;
    const int kh = warp % a.Hkv, bt = warp / a.Hkv, b = bt / T, t = bt % T;
    const int bg = b * a.Hkv + kh;
    const int pos = a.len[b] - T + t - (base ? base[b] : 0);
    if (pos < 0 || pos >= a.cap) return;
    store_row(a, bg, pos, warp, lane);   // warp = (b*T + t)*Hkv + kh: the row of the (B, T, Hkv, D) input
}

// window rows of one request: k, v (Hkv, w, D) -> win[(g*Wcap + j)], avg (Hkv, D) -> avg_k, win_len[request] = w
__global__ void window_fill_kernel(const uint4 *__restrict__ k, const uint4 *__restrict__ v, const uint4 *__restrict__ avg,
                                   uint4 *__restrict__ win, uint4 *__restrict__ avg_store, int32_t *win_len_b, int Hkv, int w,
                                   int Wcap) {
    const int total = Hkv * w * 32;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
        const int chunk = t & 31, row = t >> 5;
        const int g = row / w, j = row % w;
        const uint4 val = (chunk < 16) ? k[(size_t)row * 16 + chunk] : v[(size_t)row * 16 + chunk - 16];
        win[((size_t)g * Wcap + j) * 32 + chunk] = val;
    }
    const int gt = blockIdx.x * blockDim.x + threadIdx.x;
    if (gt < Hkv * 16) avg_store[gt] = avg[gt];
    if (gt == 0) *win_len_b = w;
}

int launch_simhash(mpig_ctx *ctx, const void *query_bf16, int32_t *codes, float *qnorm, const AppendParams *ap,
                   cudaStream_t s, bool pdl, int rows) {
    MPIG_REQUIRE(ctx->hash_func_set, MPIG_ESTATE, "SimHash before mpig_set_hash_func: the projection has not been set");
    const int K = ctx->cfg.K, L = ctx->cfg.L;
    const int H = rows > 0 ? rows : ctx->H;
    const int n_hash = (L + SH_TABLES - 1) / SH_TABLES;
    AppendParams a = {};
    if (ap) a = *ap;
    const int grid = n_hash + ((ap && ap->k_new) ? 1 : 0);
    const size_t smem = (size_t)SH_MBLOCK * SH_D * 2 + (size_t)(SH_MBLOCK + SH_TABLES * K) * SH_STRIDE * 2 +
                        (size_t)SH_MBLOCK * SH_TABLES * K + 16;
    MPIG_FUNC_ATTR(simhash_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid, (H + SH_MBLOCK - 1) / SH_MBLOCK);
    cfg.blockDim = dim3(SH_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    MPIG_CUDA(cudaLaunchKernelEx(&cfg, simhash_kernel, (const __nv_bfloat16 *)query_bf16,
                                 (const __nv_bfloat16 *)ctx->hash_func_t, codes, qnorm, H, K, L, n_hash, a));
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

int launch_append_tokens(mpig_ctx *ctx, const AppendParams &ap, int T, cudaStream_t s, const int32_t *base) {
    const int warps = ap.BG * T;
    append_tokens_kernel<<<(warps + 7) / 8, 256, 0, s>>>(ap, T, base);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

}  // namespace mpig

using namespace mpig;

extern "C" {

int mpig_simhash(mpig_ctx *ctx, const void *query_bf16, int32_t *codes, float *query_norm, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx && query_bf16 && codes, MPIG_EINVAL, "mpig_simhash: null argument");
    return launch_simhash(ctx, query_bf16, codes, query_norm, nullptr, as_stream(stream), false);
}

int mpig_window_fill(mpig_ctx *ctx, int layer, int request, const void *avg_k_bf16, const void *k_bf16, const void *v_bf16,
                     int w, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_window_fill");
    if (rc) return rc;
    MPIG_REQUIRE(request >= 0 && request < ctx->cfg.batch_size, MPIG_EINVAL, "mpig_window_fill: request %d out of range", request);
    MPIG_REQUIRE(w >= 0 && w <= ctx->Wcap, MPIG_EINVAL, "mpig_window_fill: w=%d exceeds window capacity %d", w, ctx->Wcap);
    MPIG_REQUIRE(avg_k_bf16 && (w == 0 || (k_bf16 && v_bf16)), MPIG_EINVAL, "mpig_window_fill: null input");
    const LayerStore &ls = ctx->layers[layer];
    const int Hkv = ctx->cfg.num_key_value_heads;
    uint4 *win = reinterpret_cast<uint4 *>(ls.win + (size_t)request * Hkv * ctx->Wcap * ctx->rec_bytes);
    uint4 *avg = reinterpret_cast<uint4 *>(ls.avg_k + (size_t)request * Hkv * ctx->cfg.head_dim);
    const int total = std::max(Hkv * w * 32, Hkv * 16);
    window_fill_kernel<<<(total + 255) / 256, 256, 0, as_stream(stream)>>>((const uint4 *)k_bf16, (const uint4 *)v_bf16,
                                                                          (const uint4 *)avg_k_bf16, win, avg,
                                                                          ctx->win_len + request, Hkv, w, ctx->Wcap);
    MPIG_LAUNCH_CHECK(ctx);
    ctx->h_win_len[request] = w;   // every sparse layer of a request is filled with the same w (attnserver.py:128-153)
    return MPIG_OK;
}

}  // extern "C"
