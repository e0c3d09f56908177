// aux_ops.cu -- harness-side fused elementwise kernels (see include/magicpig_b200_aux.h).  Not the hot path.
#include "../../include/magicpig_b200_aux.h"
#include "common.cuh"

namespace mpig {

__device__ __forceinline__ void unpack8(const uint4 &v, float f[8]) {
    f[0] = bf16lo(v.x); f[1] = bf16hi(v.x); f[2] = bf16lo(v.y); f[3] = bf16hi(v.y);
    f[4] = bf16lo(v.z); f[5] = bf16hi(v.z); f[6] = bf16lo(v.w); f[7] = bf16hi(v.w);
}
__device__ __forceinline__ uint4 pack8(const float f[8]) {
    uint4 v;
    v.x = (uint32_t)f32_to_bf16_rne(f[0]) | ((uint32_t)f32_to_bf16_rne(f[1]) << 16);
    v.y = (uint32_t)f32_to_bf16_rne(f[2]) | ((uint32_t)f32_to_bf16_rne(f[3]) << 16);
    v.z = (uint32_t)f32_to_bf16_rne(f[4]) | ((uint32_t)f32_to_bf16_rne(f[5]) << 16);
    v.w = (uint32_t)f32_to_bf16_rne(f[6]) | ((uint32_t)f32_to_bf16_rne(f[7]) << 16);
    return v;
}

// one CTA per row; each thread owns up to 2 chunks of 8 elements (hidden <= 16 * blockDim)
__global__ void __launch_bounds__(512) add_rmsnorm_kernel(uint4 *__restrict__ h, const uint4 *__restrict__ delta,
                                                          const uint4 *__restrict__ w, float eps, uint4 *__restrict__ x, int hidden) {
    __shared__ float red[32];
    const int row = blockIdx.x, nchunk = hidden / 8;
    uint4 *hr = h + (size_t)row * nchunk;
    float vals[2][8];
    float ss = 0.f;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int c = threadIdx.x + r * blockDim.x;
        if (c < nchunk) {
            unpack8(hr[c], vals[r]);
            if (delta) {
                float dv[8];
                unpack8(delta[(size_t)row * nchunk + c], dv);
#pragma unroll
                for (int i = 0; i < 8; ++i) vals[r][i] = bf16_bits_to_f32(f32_to_bf16_rne(vals[r][i] + dv[i]));  // residual stream is bf16
                hr[c] = pack8(vals[r]);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) ss += vals[r][i] * vals[r][i];
        }
    }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x < 32) {
        float t = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
        t = warp_sum(t);
        if (threadIdx.x == 0) red[0] = rsqrtf(t / (float)hidden + eps);
    }
    __syncthreads();
    const float inv = red[0];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int c = threadIdx.x + r * blockDim.x;
        if (c < nchunk) {
            float wv[8], o[8];
            unpack8(w[c], wv);
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i] = vals[r][i] * inv * wv[i];
            x[(size_t)row * nchunk + c] = pack8(o);
        }
    }
}

// grid (Hq + 2*Hkv, B), 64 threads: thread t owns the rotation pair (t, t + 64) of one head
__global__ void rope_split_kernel(const __nv_bfloat16 *__restrict__ qkv, const __nv_bfloat16 *__restrict__ cos_tab,
                                  const __nv_bfloat16 *__restrict__ sin_tab, const int64_t *__restrict__ pos,
                                  __nv_bfloat16 *__restrict__ q_out, __nv_bfloat16 *__restrict__ k_out,
                                  __nv_bfloat16 *__restrict__ v_out, int Hq, int Hkv) {
    constexpr int d = 128;
    pdl_launch_dependents();  // the consumer (simhash) may start its constant-data prologue; it waits for this grid before reading q/k/v
    const int hd = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
    const __nv_bfloat16 *src = qkv + ((size_t)b * (Hq + 2 * Hkv) + hd) * d;
    __nv_bfloat16 *dst;
    bool rot = true;
    if (hd < Hq) dst = q_out + ((size_t)b * Hq + hd) * d;
    else if (hd < Hq + Hkv) dst = k_out + ((size_t)b * Hkv + (hd - Hq)) * d;
    else {
        dst = v_out + ((size_t)b * Hkv + (hd - Hq - Hkv)) * d;
        rot = false;
    }
    const float x1 = __bfloat162float(src[t]), x2 = __bfloat162float(src[t + 64]);
    if (!rot) {
        dst[t] = src[t];
        dst[t + 64] = src[t + 64];
        return;
    }
    const int64_t p = pos[b];
    const float c1 = __bfloat162float(cos_tab[p * d + t]), s1 = __bfloat162float(sin_tab[p * d + t]);
    const float c2 = __bfloat162float(cos_tab[p * d + t + 64]), s2 = __bfloat162float(sin_tab[p * d + t + 64]);
    // x * cos + rotate_half(x) * sin,  rotate_half(x) = cat(-x2, x1)   (models/utils.py:36-44)
    dst[t] = __float2bfloat16_rn(x1 * c1 - x2 * s1);
    dst[t + 64] = __float2bfloat16_rn(x2 * c2 + x1 * s2);
}

__global__ void silu_mul_kernel(const uint4 *__restrict__ gu, uint4 *__restrict__ out, int rows, int inter) {
    const int nchunk = inter / 8;
    const size_t total = (size_t)rows * nchunk;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const size_t row = t / nchunk, c = t % nchunk;
        float g[8], u[8], o[8];
        unpack8(gu[row * 2 * nchunk + c], g);
        unpack8(gu[row * 2 * nchunk + nchunk + c], u);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = (g[i] / (1.f + __expf(-g[i]))) * u[i];
        out[t] = pack8(o);
    }
}

}  // namespace mpig

using namespace mpig;

extern "C" {

int mpig_aux_add_rmsnorm(void *h_inout, const void *delta, const void *weight, float eps, void *x_out, int rows, int hidden,
                         void *stream) {
    MPIG_REQUIRE(h_inout && weight && x_out && rows > 0 && hidden > 0 && hidden % 8 == 0 && hidden <= 16 * 512, MPIG_EINVAL,
                 "mpig_aux_add_rmsnorm: bad arguments (hidden=%d)", hidden);
    add_rmsnorm_kernel<<<rows, 512, 0, as_stream(stream)>>>((uint4 *)h_inout, (const uint4 *)delta, (const uint4 *)weight, eps,
                                                           (uint4 *)x_out, hidden);
    MPIG_CUDA(cudaGetLastError());
    return MPIG_OK;
}

int mpig_aux_rope_split(const void *qkv, const void *cos_tab, const void *sin_tab, const int64_t *pos, void *q_out, void *k_out,
                        void *v_out, int B, int Hq, int Hkv, void *stream) {
    MPIG_REQUIRE(qkv && cos_tab && sin_tab && pos && q_out && k_out && v_out && B > 0, MPIG_EINVAL, "mpig_aux_rope_split: bad arguments");
    rope_split_kernel<<<dim3(Hq + 2 * Hkv, B), 64, 0, as_stream(stream)>>>(
        (const __nv_bfloat16 *)qkv, (const __nv_bfloat16 *)cos_tab, (const __nv_bfloat16 *)sin_tab, pos, (__nv_bfloat16 *)q_out,
        (__nv_bfloat16 *)k_out, (__nv_bfloat16 *)v_out, Hq, Hkv);
    MPIG_CUDA(cudaGetLastError());
    return MPIG_OK;
}

int mpig_aux_silu_mul(const void *gate_up, void *out, int rows, int inter, void *stream) {
    MPIG_REQUIRE(gate_up && out && rows > 0 && inter > 0 && inter % 8 == 0, MPIG_EINVAL, "mpig_aux_silu_mul: bad arguments");
    const size_t total = (size_t)rows * inter / 8;
    int dev = 0, sms = 0;
    MPIG_CUDA(cudaGetDevice(&dev));
    MPIG_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)sms * 8);   // grid-stride: 8 blocks per SM
    silu_mul_kernel<<<blocks, 256, 0, as_stream(stream)>>>((const uint4 *)gate_up, (uint4 *)out, rows, inter);
    MPIG_CUDA(cudaGetLastError());
    return MPIG_OK;
}

}  // extern "C"
