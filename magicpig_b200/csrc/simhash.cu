// simhash.cu -- stage 1: SimHash of the decode queries, plus the small per-step window maintenance.
//
// Replaces the GPU-side torch glue of LSHSparseAttnServer.decode:
//   attnserver.py:264-270   norm_q = q/||q|| (bf16) ; P = norm_q @ hash_func ; bit = P > 0 ;
//                           code[h,l] = sum_i bit[h, l*K+i] << i                 -> simhash_kernel
//   attnserver.py:300       ||q||_2 in fp32 of the bf16 query                     -> same kernel
//   attnserver.py:275-290   k_new -= avg_k ; append k_new, v_new to the window    -> same launch (extra CTA)
//   attnserver.py:196-198   plan(): kv_last_page_len += 1                         -> plan_kernel
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


__device__ __forceinline__ void append_rows(const AppendParams &a) {
    // one warp per (b, g): 256 B of K (centred, bf16 arithmetic as torch: fp32 subtract, RNE) + 256 B of V
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
    for (int bg = warp; bg < a.BG; bg += warps) {
        const int b = bg / a.Hkv;
        const int pos = a.len[b] - 1;
        if (pos < 0 || pos >= a.cap) continue;
        uint8_t *rec = a.rows + ((size_t)bg * a.cap + pos) * (4 * SH_D);
        const uint2 kk = *reinterpret_cast<const uint2 *>(a.k_new + (size_t)bg * SH_D + 4 * lane);
        uint2 ko = kk;
        if (a.avg_k) {
            const uint2 av = *reinterpret_cast<const uint2 *>(a.avg_k + (size_t)bg * SH_D + 4 * lane);
            ko.x = (uint32_t)f32_to_bf16_rne(bf16lo(kk.x) - bf16lo(av.x)) | ((uint32_t)f32_to_bf16_rne(bf16hi(kk.x) - bf16hi(av.x)) << 16);
            ko.y = (uint32_t)f32_to_bf16_rne(bf16lo(kk.y) - bf16lo(av.y)) | ((uint32_t)f32_to_bf16_rne(bf16hi(kk.y) - bf16hi(av.y)) << 16);
        }
        *reinterpret_cast<uint2 *>(rec + 8 * lane) = ko;
        *reinterpret_cast<uint2 *>(rec + 2 * SH_D + 8 * lane) =
            *reinterpret_cast<const uint2 *>(a.v_new + (size_t)bg * SH_D + 4 * lane);
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

__global__ void append_kernel(AppendParams ap) { append_rows(ap); }

// T new rows per (request, kv-head) of a verification step: one warp per (b, t, kv-head), the same bf16 arithmetic as
// append_rows.  k_new / v_new are (B, T, Hkv, D); row t of request b goes to position len[b] - T + t (len already advanced by
// mpig_plan_tokens).  The attention launch that reads the rows follows under programmatic dependent launch.
__global__ void append_tokens_kernel(AppendParams a, int T) {
    pdl_launch_dependents();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= a.BG * T) return;
    const int kh = warp % a.Hkv, bt = warp / a.Hkv, b = bt / T, t = bt % T;
    const int bg = b * a.Hkv + kh;
    const int pos = a.len[b] - T + t;
    if (pos < 0 || pos >= a.cap) return;
    uint8_t *rec = a.rows + ((size_t)bg * a.cap + pos) * (4 * SH_D);
    const size_t src = (size_t)warp * SH_D + 4 * lane;   // warp = (b*T + t)*Hkv + kh: the row of the (B, T, Hkv, D) input
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

// mpig_rewind: both lengths of request b shrink by drop[b] in [0, T]; any other drop leaves the request untouched and raises bit 2
// of the context's error flags.  apply = 0: only the flag (an eager call that refuses changes no length).
__global__ void rewind_kernel(const int32_t *drop, int32_t *win_len, int32_t *dense_len, int32_t *err_flag, int B, int T, int apply) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B) {
        const int d = drop[b];
        if (d < 0 || d > T) {
            atomicOr(err_flag, 4);
            return;
        }
        if (!apply) return;
        win_len[b] = max(win_len[b] - d, 0);
        dense_len[b] = max(dense_len[b] - d, 0);
    }
}

// Lengths advance by T (1 for mpig_plan) and saturate at the capacity (the append then overwrites the last row); saturation of a
// store that is in use raises the context's device error flag (bit 0: sparse window = generation_buffer exhausted, bit 1: dense
// cache = max_length exhausted), readable with mpig_error_flags -- the host-side check in mpig_plan cannot see replays of a
// captured graph.
// The step's node records go to step_buf: the bases (lengths after the plan minus T), the parents and the ancestor masks (bit j of
// mask t: node j is node t or one of its ancestors).  parents == null: a chain (node t's parent is t - 1).  A malformed tree
// (parents[b][0] != -1 or parents[b][t] outside [0, t)) raises bit 3 and request b runs as a chain.  apply = 0: only that check
// (an eager mpig_plan_tree that refuses changes nothing).
__global__ void plan_kernel(int32_t *win_len, int32_t *dense_len, int32_t *err_flag, int B, int T, int wcap, int dcap,
                            int has_window, int has_dense, int32_t *step_buf, const int32_t *parents, int apply) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B) {
        int par[TREE_MAX];
        bool ok = true;
        for (int t = 0; t < T; ++t) {
            par[t] = parents ? parents[b * T + t] : t - 1;
            ok &= (t == 0) ? (par[t] == -1) : (par[t] >= 0 && par[t] < t);
        }
        if (!ok) {
            atomicOr(err_flag, 8);
            for (int t = 0; t < T; ++t) par[t] = t - 1;
        }
        if (!apply) return;
        int w = win_len[b] + T, dl = dense_len[b] + T;
        if (w > wcap) {
            w = wcap;
            if (has_window) atomicOr(err_flag, 1);
        }
        if (dl > dcap) {
            dl = dcap;
            if (has_dense) atomicOr(err_flag, 2);
        }
        win_len[b] = w;
        dense_len[b] = dl;
        int32_t *bases = step_bases(step_buf, B), *masks = step_masks(step_buf) + b * T, *pout = step_parents(step_buf, B) + b * T;
        bases[2 * b] = w - T;
        bases[2 * b + 1] = dl - T;
        uint32_t m[TREE_MAX];
        for (int t = 0; t < T; ++t) {
            m[t] = (t > 0 ? m[par[t]] : 0u) | (1u << t);
            masks[t] = (int32_t)m[t];
            pout[t] = par[t];
        }
    }
}

// mpig_accept: per request b, the root path nodes[b][0..count[b]) of the pending step becomes the step's first count[b] rows.  One
// warp per (row-owning layer, request, kv-head); lane l moves 16-byte chunk l (+32, ...) of each record, and reads every chunk of
// the path before it writes any, so the in-place move needs no staging.  A path is valid when 0 <= count <= T, nodes[0] = 0 and
// parents[nodes[i]] = nodes[i-1]; an invalid one leaves request b untouched and raises bit 3.  Rows are addressed from the step
// bases plan_kernel recorded (never from the lengths this kernel rewrites) and stay inside each store's capacity.  The warp of
// (table entry 0, b, kv-head 0) sets both lengths to base + count.  apply = 0: only the check.
__global__ void __launch_bounds__(256) accept_path_kernel(const AcceptLayer *layers, int n_layers, const int32_t *nodes,
                                                          const int32_t *count, const int32_t *step_buf, int32_t *win_len,
                                                          int32_t *dense_len, int32_t *err_flag, int B, int Hkv, int T, int rec16,
                                                          int apply) {
    const int wid = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    const int nl = max(n_layers, 1);
    if (wid >= nl * B * Hkv) return;
    const int li = wid / (B * Hkv), b = (wid / Hkv) % B, head = wid % Hkv;
    const int32_t *par = step_parents(step_buf, B) + b * T;
    const int cnt = count[b];
    bool ok = cnt >= 0 && cnt <= T;
    int nd[TREE_MAX];
#pragma unroll
    for (int i = 0; i < TREE_MAX; ++i) {
        nd[i] = i;
        if (ok && i < cnt) {
            const int n = nodes[b * T + i];
            if (i == 0) ok = (n == 0);
            else ok = (n > 0 && n < T && par[n] == nd[i - 1]);
            nd[i] = n;
        }
    }
    const bool leader = (li == 0 && head == 0);
    if (!ok) {
        if (leader && lane == 0) atomicOr(err_flag, 8);
        return;
    }
    if (!apply) return;
    const int32_t *bases = step_bases(step_buf, B);
    if (li < n_layers) {
        const AcceptLayer ly = layers[li];
        const int base = bases[2 * b + ly.dense];
        uint4 *rows = reinterpret_cast<uint4 *>(ly.rows + ((size_t)b * Hkv + head) * (size_t)ly.cap * rec16 * 16);
        for (int ch = lane; ch < rec16; ch += 32) {
            uint4 v[TREE_MAX];
#pragma unroll
            for (int i = 0; i < TREE_MAX; ++i) {
                const int src = base + nd[i];
                if (i < cnt && nd[i] != i && base + i >= 0 && src < ly.cap) v[i] = rows[(size_t)src * rec16 + ch];
            }
#pragma unroll
            for (int i = 0; i < TREE_MAX; ++i) {
                const int src = base + nd[i];
                if (i < cnt && nd[i] != i && base + i >= 0 && src < ly.cap) rows[(size_t)(base + i) * rec16 + ch] = v[i];
            }
        }
    }
    if (leader && lane == 0) {
        win_len[b] = max(bases[2 * b] + cnt, 0);
        dense_len[b] = max(bases[2 * b + 1] + cnt, 0);
    }
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

int launch_append(mpig_ctx *ctx, const AppendParams &ap, cudaStream_t s) {
    append_kernel<<<1, 256, 0, s>>>(ap);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

int launch_append_tokens(mpig_ctx *ctx, const AppendParams &ap, int T, cudaStream_t s) {
    const int warps = ap.BG * T;
    append_tokens_kernel<<<(warps + 7) / 8, 256, 0, s>>>(ap, T);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

// the host-mirror checks of mpig_plan for a step of T tokens (nothing is modified when one fails)
static int plan_checks(mpig_ctx *ctx, int T, bool has_window, bool has_dense, const char *who) {
    for (int b = 0; b < ctx->cfg.batch_size; ++b) {
        MPIG_REQUIRE(!has_window || ctx->h_win_len[b] + T <= ctx->Wcap, MPIG_ESTATE,
                     "%s: request %d: the sparse window is full (%d rows = sink + local + generation_buffer); "
                     "raise generation_buffer or clear()", who, b, ctx->Wcap);
        MPIG_REQUIRE(!has_dense || ctx->h_dense_len[b] == 0 || ctx->h_dense_len[b] + T <= ctx->cfg.max_length, MPIG_ESTATE,
                     "%s: request %d: the dense KV cache is full (max_length = %d)", who, b, ctx->cfg.max_length);
    }
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

// mpig_plan / mpig_plan_tokens / mpig_plan_tree: the host-mirror checks (exact until a plan is captured into a CUDA graph: replays
// advance only the device side), then every length advances by T on the device and the step's node records are written
static int plan_step(mpig_ctx *ctx, int T, cudaStream_t s, const char *who, const int32_t *parents = nullptr) {
    const int B = ctx->cfg.batch_size;
    int has_window = 0, has_dense = 0;
    for (const auto &ls : ctx->layers) {
        has_window |= (ls.sparse && ctx->Wcap > 0);
        has_dense |= (ls.dense && ls.dense_kv != nullptr);
    }
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    MPIG_CUDA(cudaStreamIsCapturing(s, &cap));
    if (cap != cudaStreamCaptureStatusNone) {
        ctx->h_len_exact = false;
        ctx->plan_captured = true;
    }
    if (ctx->h_len_exact) {
        const int rc = plan_checks(ctx, T, has_window, has_dense, who);
        if (rc) return rc;
        for (int b = 0; b < B; ++b) {
            ctx->h_win_len[b] = std::min(ctx->h_win_len[b] + T, ctx->Wcap);
            ctx->h_dense_len[b] = std::min(ctx->h_dense_len[b] + T, ctx->cfg.max_length);
        }
    }
    plan_kernel<<<(B + 127) / 128, 128, 0, s>>>(ctx->win_len, ctx->dense_len, ctx->err_flag, B, T, ctx->Wcap, ctx->cfg.max_length,
                                               has_window, has_dense, ctx->step_buf, parents, 1);
    MPIG_LAUNCH_CHECK(ctx);
    ctx->pending_T = T;
    ctx->rewound = false;
    ctx->pending_tree = (parents != nullptr);
    return MPIG_OK;
}

// host restatement of the device checks (eager calls refuse before anything is modified)
static bool tree_ok(const int32_t *par, int T) {
    for (int t = 0; t < T; ++t)
        if ((t == 0) ? (par[t] != -1) : (par[t] < 0 || par[t] >= t)) return false;
    return true;
}
static bool path_ok(const int32_t *nodes, int cnt, const int32_t *par, int T) {
    if (cnt < 0 || cnt > T) return false;
    for (int i = 0; i < cnt; ++i) {
        const int n = nodes[i];
        if (i == 0 ? (n != 0) : (n <= 0 || n >= T || par[n] != nodes[i - 1])) return false;
    }
    return true;
}

static int launch_accept(mpig_ctx *ctx, const int32_t *nodes, const int32_t *count, int T, int apply, cudaStream_t s) {
    const int B = ctx->cfg.batch_size, Hkv = ctx->cfg.num_key_value_heads;
    const int warps = std::max(ctx->n_accept_layers, 1) * B * Hkv;
    accept_path_kernel<<<(warps + 7) / 8, 256, 0, s>>>((const AcceptLayer *)ctx->accept_layers, ctx->n_accept_layers, nodes, count,
                                                       ctx->step_buf, ctx->win_len, ctx->dense_len, ctx->err_flag, B, Hkv, T,
                                                       ctx->rec_bytes / 16, apply);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

// the device lengths are the truth after an eager rewind / accept: the host mirror follows them, so the eager checks of mpig_plan
// stay exact
static int refresh_len_mirror(mpig_ctx *ctx, cudaStream_t s) {
    const int B = ctx->cfg.batch_size;
    std::vector<int32_t> wl(B), dl(B);
    MPIG_CUDA(cudaMemcpyAsync(wl.data(), ctx->win_len, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    MPIG_CUDA(cudaMemcpyAsync(dl.data(), ctx->dense_len, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    MPIG_CUDA(cudaStreamSynchronize(s));
    for (int b = 0; b < B; ++b) {
        ctx->h_win_len[b] = wl[b];
        ctx->h_dense_len[b] = dl[b];
    }
    return MPIG_OK;
}

int mpig_plan(mpig_ctx *ctx, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "mpig_plan: null context");
    return plan_step(ctx, 1, as_stream(stream), "mpig_plan");
}

int mpig_plan_tokens(mpig_ctx *ctx, int T, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "mpig_plan_tokens: null context");
    MPIG_REQUIRE(T >= 1 && T <= ctx->tok_max, MPIG_EINVAL,
                 "mpig_plan_tokens: T=%d outside [1, %d] (mpig_reserve_query_tokens sets the upper bound)", T, ctx->tok_max);
    return plan_step(ctx, T, as_stream(stream), "mpig_plan_tokens");
}

int mpig_rewind(mpig_ctx *ctx, const int32_t *drop, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx && drop, MPIG_EINVAL, "mpig_rewind: null argument");
    MPIG_REQUIRE(ctx->pending_T > 0 && !ctx->rewound, MPIG_ESTATE,
                 "mpig_rewind: at most one rewind or accept per plan (no plan since the last one)");
    MPIG_REQUIRE(!ctx->pending_tree, MPIG_ESTATE, "mpig_rewind: the pending step is a tree (mpig_plan_tree); commit a path with mpig_accept");
    const int B = ctx->cfg.batch_size;
    cudaStream_t s = as_stream(stream);
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    MPIG_CUDA(cudaStreamIsCapturing(s, &cap));
    const bool eager = (cap == cudaStreamCaptureStatusNone);
    const int T = ctx->pending_T;
    if (!eager) {
        rewind_kernel<<<(B + 127) / 128, 128, 0, s>>>(drop, ctx->win_len, ctx->dense_len, ctx->err_flag, B, T, 1);
        MPIG_LAUNCH_CHECK(ctx);
        ctx->rewound = true;
        ctx->h_len_exact = false;
        return MPIG_OK;
    }
    // eager: the drops are checked first, so a refused call changes no length (only error flag bit 2 is raised) and may be
    // repeated with valid drops
    std::vector<int32_t> dh(B);
    MPIG_CUDA(cudaMemcpyAsync(dh.data(), drop, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    MPIG_CUDA(cudaStreamSynchronize(s));
    bool bad = false;
    for (int b = 0; b < B; ++b) bad |= (dh[b] < 0 || dh[b] > T);
    rewind_kernel<<<(B + 127) / 128, 128, 0, s>>>(drop, ctx->win_len, ctx->dense_len, ctx->err_flag, B, T, bad ? 0 : 1);
    MPIG_LAUNCH_CHECK(ctx);
    MPIG_REQUIRE(!bad, MPIG_EINVAL, "mpig_rewind: a drop outside [0, %d]; nothing was changed (error flag bit 2)", T);
    ctx->rewound = true;
    return refresh_len_mirror(ctx, s);
}

int mpig_plan_tree(mpig_ctx *ctx, int T, const int32_t *parents, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx && parents, MPIG_EINVAL, "mpig_plan_tree: null argument");
    MPIG_REQUIRE(T >= 1 && T <= ctx->tok_max, MPIG_EINVAL,
                 "mpig_plan_tree: T=%d outside [1, %d] (mpig_reserve_query_tokens sets the upper bound)", T, ctx->tok_max);
    const int B = ctx->cfg.batch_size;
    cudaStream_t s = as_stream(stream);
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    MPIG_CUDA(cudaStreamIsCapturing(s, &cap));
    if (cap == cudaStreamCaptureStatusNone) {
        // eager: the trees are checked first, so a refused call changes nothing (only error flag bit 3 is raised)
        std::vector<int32_t> ph((size_t)B * T);
        MPIG_CUDA(cudaMemcpyAsync(ph.data(), parents, ph.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
        MPIG_CUDA(cudaStreamSynchronize(s));
        bool bad = false;
        for (int b = 0; b < B; ++b) bad |= !tree_ok(ph.data() + (size_t)b * T, T);
        if (bad) {
            plan_kernel<<<(B + 127) / 128, 128, 0, s>>>(ctx->win_len, ctx->dense_len, ctx->err_flag, B, T, ctx->Wcap,
                                                       ctx->cfg.max_length, 0, 0, ctx->step_buf, parents, 0);
            MPIG_LAUNCH_CHECK(ctx);
            set_error("mpig_plan_tree: a malformed tree (parents[b][0] must be -1 and 0 <= parents[b][t] < t); nothing was changed "
                      "(error flag bit 3)");
            return MPIG_EINVAL;
        }
    }
    return plan_step(ctx, T, s, "mpig_plan_tree", parents);
}

int mpig_accept(mpig_ctx *ctx, const int32_t *nodes, const int32_t *count, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx && nodes && count, MPIG_EINVAL, "mpig_accept: null argument");
    MPIG_REQUIRE(ctx->pending_T > 0 && !ctx->rewound, MPIG_ESTATE,
                 "mpig_accept: at most one rewind or accept per plan (no plan since the last one)");
    const int B = ctx->cfg.batch_size, T = ctx->pending_T;
    cudaStream_t s = as_stream(stream);
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    MPIG_CUDA(cudaStreamIsCapturing(s, &cap));
    if (cap != cudaStreamCaptureStatusNone) {
        const int rc = launch_accept(ctx, nodes, count, T, 1, s);
        if (rc) return rc;
        ctx->rewound = true;
        ctx->h_len_exact = false;
        return MPIG_OK;
    }
    // eager: the paths are checked against the step's parents first, so a refused call changes nothing and may be repeated
    std::vector<int32_t> nh((size_t)B * T), ch(B), ph((size_t)B * T);
    MPIG_CUDA(cudaMemcpyAsync(nh.data(), nodes, nh.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    MPIG_CUDA(cudaMemcpyAsync(ch.data(), count, ch.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    MPIG_CUDA(cudaMemcpyAsync(ph.data(), step_parents(ctx->step_buf, B), ph.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    MPIG_CUDA(cudaStreamSynchronize(s));
    bool bad = false;
    for (int b = 0; b < B; ++b) bad |= !path_ok(nh.data() + (size_t)b * T, ch[b], ph.data() + (size_t)b * T, T);
    const int rc = launch_accept(ctx, nodes, count, T, bad ? 0 : 1, s);
    if (rc) return rc;
    MPIG_REQUIRE(!bad, MPIG_EINVAL,
                 "mpig_accept: a path that is not a root path of the pending step (count outside [0, %d], nodes[0] != 0 or "
                 "parents[nodes[i]] != nodes[i-1]); nothing was changed (error flag bit 3)", T);
    ctx->rewound = true;
    return refresh_len_mirror(ctx, s);
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
