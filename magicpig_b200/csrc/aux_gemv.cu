// aux_gemv.cu -- harness-side weight-streaming GEMV for the decode step (see include/magicpig_b200_aux.h).  Not the hot path.
//
// At decode batch sizes (B <= 8 tokens) the model's linear layers (models/llama.py:195-218: q/k/v, o, gate/up, down) are
// matrix-vector products whose whole cost is streaming the bf16 weights out of HBM once.  The library GEMM tiles torch picks
// for M = 1 reach 2-3.5 TB/s on the smaller matrices (34-50 MB: a few waves of large tiles, split-K with a second reduce
// kernel); this kernel is organised around the stream instead:
//   * a warp owns R = 2 output rows at a time; a lane reads 16 B (8 bf16) of each row per step, 32 lanes = one 512-B line
//     segment per row, UN steps (UN x R 16-B loads per lane) in flight before the first FMA;
//   * x (B x K bf16, <= 115 KB) is staged once per CTA in shared memory and read as conflict-free 16-B vectors;
//   * fp32 accumulation, one shuffle reduction per row at the end, bf16 (RNE) out;
//   * optional fused SwiGLU epilogue: with W = [gate; up] the warp computes row i of both halves and writes
//     silu(gate_i) * up_i directly, so the (B, 2*inter) intermediate and the silu_mul launch disappear;
//   * optional fused prologue: x = rmsnorm(h + delta) * w computed by every CTA while it stages x (the residual stream is
//     ping-ponged: CTA 0 writes h + delta to a second buffer), which removes the add_rmsnorm launch in front of the q/k/v and
//     gate/up projections;
//   * optional fused RoPE epilogue for the q/k/v projection: a warp owns the output pair (t, t + 64) of one head, rotates it
//     (models/utils.py:36-44) and writes q / k / v in the layout the attention server takes, which removes rope_split.
#include "../../include/magicpig_b200_aux.h"
#include "common.cuh"

namespace mpig {

constexpr int GV_THREADS = 256;
constexpr int GV_R = 2;    // rows per warp per pass
constexpr int GV_UN = 4;   // k-steps in flight

__device__ __forceinline__ uint4 ldg_stream16(const uint4 *p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void unpack8f(const uint4 &v, float f[8]) {
    f[0] = bf16lo(v.x); f[1] = bf16hi(v.x); f[2] = bf16lo(v.y); f[3] = bf16hi(v.y);
    f[4] = bf16lo(v.z); f[5] = bf16hi(v.z); f[6] = bf16lo(v.w); f[7] = bf16hi(v.w);
}

enum { GV_PLAIN = 0, GV_SWIGLU = 1, GV_ROPE = 2 };

struct GemvArgs {
    const uint4 *W;            // (N or 2N rows, K) row-major bf16
    const uint4 *x;            // (B, K) bf16 -- PRE == false
    __nv_bfloat16 *y;          // (B, N) bf16 -- PLAIN / SWIGLU
    int N, K;
    // PRE: x = rmsnorm(h_in + delta) * lnw, h_out = h_in + delta
    const uint4 *h_in, *delta, *lnw;
    uint4 *h_out;
    float eps;
    // ROPE epilogue: N = (Hq + 2*Hkv) * 128 rows = q heads | k heads | v heads
    const __nv_bfloat16 *cos_tab, *sin_tab;
    const int64_t *pos;
    __nv_bfloat16 *q_out, *k_out, *v_out;
    int Hq, Hkv;
    int pdl;                   // bit 0: (q/k/v projection) let the next kernel -- the fused attention -- launch early;
                               // bit 1: (plain GEMV) this launch carries the PDL attribute: wait for the producer before reading x
};

static int g_aux_pdl = 0;      // mpig_aux_set_pdl

// grid = ceil(N / (8 warps * GV_R)); dynamic smem = B * K * 2 bytes.  K % 256 == 0.
template <int B, int MODE, bool PRE>
__global__ void __launch_bounds__(GV_THREADS) gemv_kernel(const __grid_constant__ GemvArgs a) {
    extern __shared__ __align__(16) uint8_t gv_smem[];
    __shared__ float red[B][GV_THREADS / 32];
    uint4 *sx = reinterpret_cast<uint4 *>(gv_smem);   // [B][K/8]
    const int N = a.N, K = a.K;
    const int kv = K >> 3;                            // 16-B vectors per row
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // Programmatic dependent launch only on the two edges around the attention kernel, and only on request (mpig_aux_set_pdl).
    // PDL on EVERY GEMV is slower: grids parked at griddepcontrol.wait hold registers / shared memory the running weight
    // stream needs.  The fused attention kernel takes a whole SM per CTA, so it cannot squat beside running GEMV CTAs:
    // triggering it early only hides its launch latency and constant-data prologue behind this kernel's tail; and the
    // o-projection that follows it parks on SMs the attention grid does not use or has already left.
    if (MODE == GV_ROPE && (a.pdl & 1)) pdl_launch_dependents();
    if (MODE == GV_PLAIN && !PRE && (a.pdl & 2)) pdl_wait();
    // the warp's output rows
    const int unit = blockIdx.x * (GV_THREADS / 32) + warp;   // pair of rows
    int rows[GV_R];
    if (MODE == GV_ROPE) {
        const int head = unit >> 6, t = unit & 63;             // (t, t + 64) of one head: the RoPE pair
        rows[0] = head * 128 + t;
        rows[1] = rows[0] + 64;
    } else {
        rows[0] = unit * GV_R;
        rows[1] = rows[0] + 1;
    }
    constexpr int NR = (MODE == GV_SWIGLU) ? 2 * GV_R : GV_R;      // weight rows streamed per pass
    const uint4 *wr[NR];
#pragma unroll
    for (int r = 0; r < GV_R; ++r) {
        const int row = min(rows[r], N - 1);
        wr[r] = a.W + (size_t)row * kv;
        if (MODE == GV_SWIGLU) wr[GV_R + r] = a.W + ((size_t)N + row) * kv;
    }
    if (!PRE) {
        for (int t = threadIdx.x; t < B * kv; t += GV_THREADS) sx[t] = a.x[t];
        __syncthreads();
    } else {
        // residual add + RMSNorm with the arithmetic of add_rmsnorm_kernel (aux_ops.cu): the sum is rounded to bf16 (it IS the
        // residual stream), the mean of squares is taken over the rounded values, the output is rounded once
        float ss[B];
#pragma unroll
        for (int b = 0; b < B; ++b) ss[b] = 0.f;
        for (int t = threadIdx.x; t < kv; t += GV_THREADS) {
#pragma unroll
            for (int b = 0; b < B; ++b) {
                float v[8];
                unpack8f(a.h_in[(size_t)b * kv + t], v);
                if (a.delta) {
                    float dv[8];
                    unpack8f(a.delta[(size_t)b * kv + t], dv);
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = bf16_bits_to_f32(f32_to_bf16_rne(v[i] + dv[i]));
                }
                uint4 pk;
                pk.x = (uint32_t)f32_to_bf16_rne(v[0]) | ((uint32_t)f32_to_bf16_rne(v[1]) << 16);
                pk.y = (uint32_t)f32_to_bf16_rne(v[2]) | ((uint32_t)f32_to_bf16_rne(v[3]) << 16);
                pk.z = (uint32_t)f32_to_bf16_rne(v[4]) | ((uint32_t)f32_to_bf16_rne(v[5]) << 16);
                pk.w = (uint32_t)f32_to_bf16_rne(v[6]) | ((uint32_t)f32_to_bf16_rne(v[7]) << 16);
                sx[(size_t)b * kv + t] = pk;   // h + delta for now
                if (blockIdx.x == 0) a.h_out[(size_t)b * kv + t] = pk;
#pragma unroll
                for (int i = 0; i < 8; ++i) ss[b] += v[i] * v[i];
            }
        }
#pragma unroll
        for (int b = 0; b < B; ++b) {
            const float w = warp_sum(ss[b]);
            if (lane == 0) red[b][warp] = w;
        }
        __syncthreads();
        float inv[B];
#pragma unroll
        for (int b = 0; b < B; ++b) {
            float t = 0.f;
#pragma unroll
            for (int w = 0; w < GV_THREADS / 32; ++w) t += red[b][w];
            inv[b] = rsqrtf(t / (float)K + a.eps);
        }
        for (int t = threadIdx.x; t < kv; t += GV_THREADS) {
            float wv[8];
            unpack8f(a.lnw[t], wv);
#pragma unroll
            for (int b = 0; b < B; ++b) {
                float v[8];
                unpack8f(sx[(size_t)b * kv + t], v);
                uint4 pk;
                pk.x = (uint32_t)f32_to_bf16_rne(v[0] * inv[b] * wv[0]) | ((uint32_t)f32_to_bf16_rne(v[1] * inv[b] * wv[1]) << 16);
                pk.y = (uint32_t)f32_to_bf16_rne(v[2] * inv[b] * wv[2]) | ((uint32_t)f32_to_bf16_rne(v[3] * inv[b] * wv[3]) << 16);
                pk.z = (uint32_t)f32_to_bf16_rne(v[4] * inv[b] * wv[4]) | ((uint32_t)f32_to_bf16_rne(v[5] * inv[b] * wv[5]) << 16);
                pk.w = (uint32_t)f32_to_bf16_rne(v[6] * inv[b] * wv[6]) | ((uint32_t)f32_to_bf16_rne(v[7] * inv[b] * wv[7]) << 16);
                sx[(size_t)b * kv + t] = pk;
            }
        }
        __syncthreads();
    }
    float acc[NR][B];
#pragma unroll
    for (int r = 0; r < NR; ++r)
#pragma unroll
        for (int b = 0; b < B; ++b) acc[r][b] = 0.f;
    if (rows[0] >= N) return;
    const int steps = kv >> 5;                         // 32 lanes x 16 B per step
    for (int s0 = 0; s0 < steps; s0 += GV_UN) {
        uint4 w[GV_UN][NR];
#pragma unroll
        for (int u = 0; u < GV_UN; ++u)
#pragma unroll
            for (int r = 0; r < NR; ++r)
                if (s0 + u < steps) w[u][r] = ldg_stream16(wr[r] + (size_t)(s0 + u) * 32 + lane);
#pragma unroll
        for (int u = 0; u < GV_UN; ++u) {
            if (s0 + u < steps) {
                float xf[B][8];
#pragma unroll
                for (int b = 0; b < B; ++b) unpack8f(sx[(size_t)b * kv + (s0 + u) * 32 + lane], xf[b]);
#pragma unroll
                for (int r = 0; r < NR; ++r) {
                    float wf[8];
                    unpack8f(w[u][r], wf);
#pragma unroll
                    for (int b = 0; b < B; ++b)
#pragma unroll
                        for (int i = 0; i < 8; ++i) acc[r][b] = fmaf(wf[i], xf[b][i], acc[r][b]);
                }
            }
        }
    }
#pragma unroll
    for (int r = 0; r < NR; ++r)
#pragma unroll
        for (int b = 0; b < B; ++b) acc[r][b] = warp_sum(acc[r][b]);
    if (lane != 0) return;
    if constexpr (MODE == GV_ROPE) {
        // q | k | v split + rotate-half RoPE on the bf16-rounded projections (what rope_split_kernel sees)
        const int head = unit >> 6, t = unit & 63;
#pragma unroll
        for (int b = 0; b < B; ++b) {
            const float x1 = bf16_bits_to_f32(f32_to_bf16_rne(acc[0][b])), x2 = bf16_bits_to_f32(f32_to_bf16_rne(acc[1][b]));
            __nv_bfloat16 *dst;
            bool rot = true;
            if (head < a.Hq) dst = a.q_out + ((size_t)b * a.Hq + head) * 128;
            else if (head < a.Hq + a.Hkv) dst = a.k_out + ((size_t)b * a.Hkv + (head - a.Hq)) * 128;
            else {
                dst = a.v_out + ((size_t)b * a.Hkv + (head - a.Hq - a.Hkv)) * 128;
                rot = false;
            }
            if (!rot) {
                dst[t] = __float2bfloat16_rn(x1);
                dst[t + 64] = __float2bfloat16_rn(x2);
            } else {
                const int64_t p = a.pos[b];
                const float c1 = __bfloat162float(a.cos_tab[p * 128 + t]), s1 = __bfloat162float(a.sin_tab[p * 128 + t]);
                const float c2 = __bfloat162float(a.cos_tab[p * 128 + t + 64]), s2 = __bfloat162float(a.sin_tab[p * 128 + t + 64]);
                dst[t] = __float2bfloat16_rn(x1 * c1 - x2 * s1);
                dst[t + 64] = __float2bfloat16_rn(x2 * c2 + x1 * s2);
            }
        }
    } else {
#pragma unroll
    for (int r = 0; r < GV_R; ++r) {
        if (rows[r] >= N) break;
#pragma unroll
        for (int b = 0; b < B; ++b) {
            float v = acc[r][b];
            if (MODE == GV_SWIGLU) {
                // both halves are rounded to bf16 first, as the unfused pair of ops would see them (models/llama.py:171-181)
                const float g = bf16_bits_to_f32(f32_to_bf16_rne(acc[r][b])), up = bf16_bits_to_f32(f32_to_bf16_rne(acc[GV_R + r][b]));
                v = (g / (1.f + __expf(-g))) * up;
            }
            a.y[(size_t)b * N + rows[r]] = __float2bfloat16_rn(v);
        }
    }
    }
}

template <int B, int MODE, bool PRE>
static int launch_gemv_t(const GemvArgs &a, cudaStream_t s) {
    const size_t smem = (size_t)B * a.K * 2;
    const int grid = (a.N + (GV_THREADS / 32) * GV_R - 1) / ((GV_THREADS / 32) * GV_R);
    MPIG_FUNC_ATTR((gemv_kernel<B, MODE, PRE>), cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(GV_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (MODE == GV_PLAIN && !PRE && (a.pdl & 2)) ? 1 : 0;
    MPIG_CUDA(cudaLaunchKernelEx(&cfg, gemv_kernel<B, MODE, PRE>, a));
    return MPIG_OK;
}
template <int B>
static int launch_gemv_b(const GemvArgs &a, int mode, bool pre, cudaStream_t s) {
    if (pre) {
        if (mode == GV_ROPE) return launch_gemv_t<B, GV_ROPE, true>(a, s);
        if (mode == GV_SWIGLU) return launch_gemv_t<B, GV_SWIGLU, true>(a, s);
        return launch_gemv_t<B, GV_PLAIN, true>(a, s);
    }
    if (mode == GV_ROPE) return launch_gemv_t<B, GV_ROPE, false>(a, s);
    if (mode == GV_SWIGLU) return launch_gemv_t<B, GV_SWIGLU, false>(a, s);
    return launch_gemv_t<B, GV_PLAIN, false>(a, s);
}
static int launch_gemv(const GemvArgs &a, int rows, int mode, bool pre, cudaStream_t s) {
    switch (rows) {
        case 1: return launch_gemv_b<1>(a, mode, pre, s);
        case 2: return launch_gemv_b<2>(a, mode, pre, s);
        case 3: return launch_gemv_b<3>(a, mode, pre, s);
        case 4: return launch_gemv_b<4>(a, mode, pre, s);
        case 5: return launch_gemv_b<5>(a, mode, pre, s);
        case 6: return launch_gemv_b<6>(a, mode, pre, s);
        case 7: return launch_gemv_b<7>(a, mode, pre, s);
        default: return launch_gemv_b<8>(a, mode, pre, s);
    }
}

}  // namespace mpig

using namespace mpig;

static int check_common(const void *weight, int rows, int N, int K, const char *who) {
    MPIG_REQUIRE(weight && rows >= 1 && rows <= 8 && N > 0 && K > 0 && K % 256 == 0, MPIG_EINVAL,
                 "%s: bad arguments (rows=%d N=%d K=%d; rows <= 8, K %% 256 == 0)", who, rows, N, K);
    MPIG_REQUIRE((size_t)rows * K * 2 <= 200 * 1024, MPIG_EUNSUPPORTED, "%s: rows*K=%d*%d does not fit in shared memory", who, rows, K);
    MPIG_REQUIRE(((uintptr_t)weight & 15) == 0, MPIG_EINVAL, "%s: weight must be 16-byte aligned", who);
    return MPIG_OK;
}

extern "C" {

int mpig_aux_gemv(const void *weight, const void *x, void *y, int rows, int N, int K, int swiglu, void *stream) {
    int rc = check_common(weight, rows, N, K, "mpig_aux_gemv");
    if (rc) return rc;
    MPIG_REQUIRE(x && y && ((uintptr_t)x & 15) == 0, MPIG_EINVAL, "mpig_aux_gemv: x / y null or x not 16-byte aligned");
    GemvArgs a = {};
    a.W = (const uint4 *)weight;
    a.x = (const uint4 *)x;
    a.y = (__nv_bfloat16 *)y;
    a.N = N;
    a.K = K;
    a.pdl = g_aux_pdl;
    return launch_gemv(a, rows, swiglu ? GV_SWIGLU : GV_PLAIN, false, as_stream(stream));
}

int mpig_aux_norm_gemv(const void *weight, const void *h_in, const void *delta, const void *ln_weight, float eps, void *h_out,
                       void *y, int rows, int N, int K, int swiglu, void *stream) {
    int rc = check_common(weight, rows, N, K, "mpig_aux_norm_gemv");
    if (rc) return rc;
    MPIG_REQUIRE(h_in && ln_weight && h_out && y && h_in != h_out, MPIG_EINVAL,
                 "mpig_aux_norm_gemv: null argument, or h_out aliases h_in (the residual stream must be ping-ponged)");
    GemvArgs a = {};
    a.W = (const uint4 *)weight;
    a.y = (__nv_bfloat16 *)y;
    a.N = N;
    a.K = K;
    a.h_in = (const uint4 *)h_in;
    a.delta = (const uint4 *)delta;
    a.lnw = (const uint4 *)ln_weight;
    a.h_out = (uint4 *)h_out;
    a.eps = eps;
    return launch_gemv(a, rows, swiglu ? GV_SWIGLU : GV_PLAIN, true, as_stream(stream));
}

int mpig_aux_norm_qkv_rope(const void *wqkv, const void *h_in, const void *delta, const void *ln_weight, float eps, void *h_out,
                           const void *cos_tab, const void *sin_tab, const int64_t *pos, void *q_out, void *k_out, void *v_out,
                           int rows, int Hq, int Hkv, int K, void *stream) {
    const int N = (Hq + 2 * Hkv) * 128;
    int rc = check_common(wqkv, rows, N, K, "mpig_aux_norm_qkv_rope");
    if (rc) return rc;
    MPIG_REQUIRE(h_in && ln_weight && h_out && h_in != h_out && cos_tab && sin_tab && pos && q_out && k_out && v_out && Hq > 0 && Hkv > 0,
                 MPIG_EINVAL, "mpig_aux_norm_qkv_rope: null argument, or h_out aliases h_in");
    GemvArgs a = {};
    a.W = (const uint4 *)wqkv;
    a.N = N;
    a.K = K;
    a.h_in = (const uint4 *)h_in;
    a.delta = (const uint4 *)delta;
    a.lnw = (const uint4 *)ln_weight;
    a.h_out = (uint4 *)h_out;
    a.eps = eps;
    a.cos_tab = (const __nv_bfloat16 *)cos_tab;
    a.sin_tab = (const __nv_bfloat16 *)sin_tab;
    a.pos = pos;
    a.q_out = (__nv_bfloat16 *)q_out;
    a.k_out = (__nv_bfloat16 *)k_out;
    a.v_out = (__nv_bfloat16 *)v_out;
    a.Hq = Hq;
    a.Hkv = Hkv;
    a.pdl = g_aux_pdl;
    return launch_gemv(a, rows, GV_ROPE, true, as_stream(stream));
}

/* bit 0: the q/k/v projection triggers programmatic launch of its successor; bit 1: plain GEMVs are launched as programmatic
 * dependents (they wait for their producer before reading x).  Process-wide; returns the previous value. */
int mpig_aux_set_pdl(int mask) {
    const int old = g_aux_pdl;
    g_aux_pdl = mask;
    return old;
}

}  // extern "C"
