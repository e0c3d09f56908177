// attend_common.cuh -- pieces shared by the gather-attention kernels (attend.cu, attend_mma.cu)
#pragma once
#include <math_constants.h>

#include "common.cuh"

namespace mpig {

constexpr int D = 128;                 // head_dim
constexpr int REC = 2 * D * 2;         // 512 B  {K row | V row}
constexpr int TILE = 32;               // rows per tile = lanes per warp
constexpr int PART_FLOATS = 4 + D;     // m, l, pad, pad, acc[128]
constexpr float LOG2E_F = 1.4426950408889634f;
constexpr int SLOT = REC + 16;         // 528 B shared-memory slot stride: 8 consecutive rows start in 8 different 16-byte bank groups

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t saddr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(saddr));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], uint32_t saddr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(saddr));
}
__device__ __forceinline__ void mma_16816(float &c0, float &c1, float &c2, float &c3, const uint32_t (&a)[4], uint32_t b0,
                                          uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c0), "+f"(c1), "+f"(c2), "+f"(c3)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    mma_16816(c[0], c[1], c[2], c[3], a, b0, b1);
}
// tickets of the last-arriver merges
__device__ __forceinline__ int atom_add_acq_rel_gpu(int *addr, int v) {
    int old;
    asm volatile("atom.acq_rel.gpu.global.add.s32 %0, [%1], %2;" : "=r"(old) : "l"(addr), "r"(v) : "memory");
    return old;
}
__device__ __forceinline__ int atom_add_acq_rel_cta_shared(int *addr, int v) {
    int old;
    asm volatile("atom.acq_rel.cta.shared.add.s32 %0, [%1], %2;" : "=r"(old) : "r"(smem_u32(addr)), "r"(v) : "memory");
    return old;
}
// x^n, 0 <= n < 2^NBITS, by repeated squaring in fp64 (error ~n_mults * 1e-16), rounded once to fp32.  The trip count is a
// compile-time constant and the multiply is predicated, so the (uniform) exponent costs no loop control: 2 * NBITS - 1 DMUL.
template <int NBITS>
__device__ __forceinline__ float ipow_f32(float x, int n) {
    double b = (double)x, r = 1.0;
#pragma unroll
    for (int i = 0; i < NBITS; ++i) {
        r = ((n >> i) & 1) ? r * b : r;
        if (i + 1 < NBITS) b *= b;
    }
    return (float)r;
}

// the same product sequence with the exponent known at compile time: no bit tests, only the multiplies that happen
// (x^149: 7 squarings + 3 products instead of 19 DMUL and ten predicates) -- bit-identical to ipow_f32<NBITS>(x, N)
template <int N>
__device__ __forceinline__ float ipow_const_f32(float x) {
    double b = (double)x, r = 1.0;
    bool first = true;
#pragma unroll
    for (int i = 0; i < 31; ++i) {
        if ((N >> i) == 0) break;
        if ((N >> i) & 1) {
            r = first ? b : r * b;
            first = false;
        }
        if ((N >> (i + 1)) != 0) b *= b;
    }
    return (float)r;
}
// importance weight of a sampled key (transform_kernel, sparse_attention.cc:173-183): returns w = 1 - (1-p)^(L-1) (L p + 1 - p),
// p = proba^K.  The two shapes of BASELINE.json get compile-time exponents; everything else the generic loop.
__device__ __forceinline__ float sample_weight(float proba, int K, int L, float Lf) {
    float pp, pw;
    if (K == 10 && L == 150) {
        pp = ipow_const_f32<10>(proba);
        pw = ipow_const_f32<149>(1.0f - pp);
    } else if (K == 11 && L == 300) {
        pp = ipow_const_f32<11>(proba);
        pw = ipow_const_f32<299>(1.0f - pp);
    } else {
        pp = ipow_f32<4>(proba, K);
        pw = ipow_f32<10>(1.0f - pp, L - 1);
    }
    const float qq = 1.0f - pp;
    return 1.0f - pw * (Lf * pp + qq);
}

// acos(x), |x| <= 1: sqrt(1 - |x|) * P7(|x|) (Abramowitz & Stegun 4.4.46, |error| <= 2e-8 rad -- below fp32 rounding of
// the result), reflected for x < 0.  ~14 instructions instead of libdevice's ~40 on the per-row critical path.
__device__ __forceinline__ float fast_acosf(float x) {
    const float a = fabsf(x);
    float pl = -0.0012624911f;
    pl = fmaf(pl, a, 0.0066700901f);
    pl = fmaf(pl, a, -0.0170881256f);
    pl = fmaf(pl, a, 0.0308918810f);
    pl = fmaf(pl, a, -0.0501743046f);
    pl = fmaf(pl, a, 0.0889789874f);
    pl = fmaf(pl, a, -0.2145988016f);
    pl = fmaf(pl, a, 1.5707963050f);
    const float r = sqrtf(1.0f - a) * pl;
    return (x >= 0.f) ? r : CUDART_PI_F - r;
}


__device__ __forceinline__ void finalize_head(const AttendParams &p, int h, float m, float l, const float acc[4], int lane) {
    // softmax_kernel :238-239 (base-2 LSE) + wv_kernel :345 (fp32 -> bf16, FBGEMM rounding)
    const float inv = (l > 0.f) ? 1.0f / l : 0.f;
    uint32_t lo = (uint32_t)f32_to_bf16_half_up(acc[0] * inv) | ((uint32_t)f32_to_bf16_half_up(acc[1] * inv) << 16);
    uint32_t hi = (uint32_t)f32_to_bf16_half_up(acc[2] * inv) | ((uint32_t)f32_to_bf16_half_up(acc[3] * inv) << 16);
    *reinterpret_cast<uint2 *>(reinterpret_cast<uint8_t *>(p.out) + ((size_t)h * D + 4 * lane) * 2) = make_uint2(lo, hi);
    if (p.out_f32)
        *reinterpret_cast<float4 *>(p.out_f32 + (size_t)h * D + 4 * lane) = make_float4(acc[0] * inv, acc[1] * inv, acc[2] * inv, acc[3] * inv);
    if (p.mve && lane == 0) {
        const float mv = m * LOG2E_F;                       // -inf when the head had no rows
        p.mve[h] = mv;
        p.mve[p.H + h] = (l > 0.f) ? log2f(l) + mv : -CUDART_INF_F;
    }
}

// Combine `n` partial states.  slot_ptr(i) returns the i-th state's base; GLOBAL selects L2 (ld.cg) reads.
// 32 states at a time: lane i fetches state i's (m, l), the warp agrees on the new max, and the 512-byte
// accumulators are then loaded four at a time (independent loads in flight).
template <bool GLOBAL, typename SlotFn>
__device__ __forceinline__ void merge_states(SlotFn slot_ptr, int n, int lane, float &M_, float &L_, float A[4]) {
    M_ = -CUDART_INF_F;
    L_ = 0.f;
    A[0] = A[1] = A[2] = A[3] = 0.f;
    for (int c0 = 0; c0 < n; c0 += 32) {
        const int cnt = min(32, n - c0);
        float m_i = -CUDART_INF_F, l_i = 0.f;
        if (lane < cnt) {
            const float *pp = slot_ptr(c0 + lane);
            m_i = GLOBAL ? __ldcg(pp) : pp[0];
            l_i = GLOBAL ? __ldcg(pp + 1) : pp[1];
        }
        const float mn = fmaxf(M_, warp_max(m_i));
        const float f_old = (M_ == -CUDART_INF_F) ? 0.f : exp2f((M_ - mn) * LOG2E_F);
        const float f_i = (m_i == -CUDART_INF_F) ? 0.f : exp2f((m_i - mn) * LOG2E_F);
        L_ = L_ * f_old + warp_sum(l_i * f_i);
#pragma unroll
        for (int i = 0; i < 4; ++i) A[i] *= f_old;
        for (int j0 = 0; j0 < cnt; j0 += 8) {   // eight 512-byte accumulators in flight
            float4 a2[8];
#pragma unroll
            for (int uu = 0; uu < 8; ++uu) {
                a2[uu] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (j0 + uu < cnt) {
                    const float4 *ap = reinterpret_cast<const float4 *>(slot_ptr(c0 + j0 + uu) + 4 + 4 * lane);
                    a2[uu] = GLOBAL ? __ldcg(ap) : *ap;
                }
            }
#pragma unroll
            for (int uu = 0; uu < 8; ++uu) {
                const float f2 = __shfl_sync(0xffffffffu, f_i, (j0 + uu) & 31);
                A[0] = fmaf(a2[uu].x, f2, A[0]);
                A[1] = fmaf(a2[uu].y, f2, A[1]);
                A[2] = fmaf(a2[uu].z, f2, A[2]);
                A[3] = fmaf(a2[uu].w, f2, A[3]);
            }
        }
        M_ = mn;
    }
}

__device__ __forceinline__ void store_state(float *part, float m, float l, const float acc[4], int lane) {
    if (lane == 0) {
        part[0] = m;
        part[1] = l;
    }
    *reinterpret_cast<float4 *>(part + 4 + 4 * lane) = make_float4(acc[0], acc[1], acc[2], acc[3]);
}


}  // namespace mpig
