// attend_prefill.cu -- prefill attention (mpig_prefill_attend): exact causal softmax attention of one sequence's query chunk over
// its keys, the operation flashinfer.prefill.single_prefill_with_kv_cache(q, k, v, causal=True, kv_layout="NHD") performs at the
// reference's prefill call site (models/llama.py:250-257).  q (q_len, Hq, d), k / v (kv_len, Hkv, d) bf16 NHD, d = 128, G = Hq / Hkv
// in [1, 8]; query i sits at position kv_len - q_len + i and sees keys [0, kv_len - q_len + i] (bottom-right alignment); scale 1/sqrt(d).
//
// A CTA owns one (kv-head h, m-block of tb = floor(128 / G) tokens).  The m-block's tb*G query rows of the kv-group are ordered
// r = t*G + g (token t0 + t, q-head h*G + g), so a row's causal limit depends on t only and every K/V tile is loaded once for the G
// heads.  That order is exactly what a 3-D TMA box (64 dims, G heads, tb tokens) of q writes, so Q comes in by TMA too; the rows
// past tb*G (at most 7) are zeroed once.  Hopper pipeline (DESIGN.md section 3.16):
//   producer        one warp of a warpgroup that hands its registers to the consumers (setmaxnreg) issues the TMA of the Q tile
//                   (two 64-dim SWIZZLE_128B atoms) and of a ring of PF_ST K/V stages of PF_KT keys, completion counted in bytes on
//                   mbarriers (full / empty per stage)
//   2 warpgroups    64 query rows each: S = Q.K^T with wgmma m64n128k16, both operands K-major in shared memory; masked online
//                   softmax in fp32 registers (the mask is skipped on tiles wholly below every row of the warp); O += P.V with P from
//                   registers as bf16 hi + lo (P rounded to plain bf16 misses 1e-3 of fp64 once a few keys take most of the
//                   probability, DESIGN.md section 3.14) and V as the MN-major B operand straight from the TMA tile; l sums the
//                   unrounded P.
// The m-blocks are launched heaviest (most keys) first.  No key splits: a short q_len is correct but uses few SMs.
#include "attend_common.cuh"
#include "gmma_common.cuh"

namespace mpig {

constexpr int PF_BM = 128;                           // query rows per CTA (two consumer warpgroups of 64)
constexpr int PF_KT = 128;                           // keys per K/V tile
constexpr int PF_ST = 2;                             // K/V stages in flight
constexpr int PF_THREADS = 384;                      // two consumer warpgroups + one producer warpgroup (one warp of it issues)
constexpr uint32_t PF_Q_ATOM = PF_BM * 128u;         // one 64-dim (128-byte) column atom of the Q tile
constexpr uint32_t PF_KV_ATOM = PF_KT * 128u;        // ... of a K or V tile
constexpr uint32_t PF_TILE = 2u * PF_KV_ATOM;        // one K or V tile (32 KB)
constexpr size_t PF_SMEM = 1024 + 2 * (size_t)PF_Q_ATOM + 2 * (size_t)PF_ST * PF_TILE + 64;

struct PrefillParams {
    __nv_bfloat16 *out;   // (q_len, Hq, D)
    float *out_f32;       // same or null
    int q_len, kv_len, Hq, Hkv, G, tb, nmb;
};

// D(64 x 128, fp32) (+)= A(64 x 16) * B(16 x 128), A and B bf16 K-major in shared memory; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_m64n128k16_ss(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
        "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// D(64 x 128, fp32) += A(64 x 16, registers: the accumulator layout of m64n16) * B(16 x 128), B bf16 MN-major in shared memory
__device__ __forceinline__ void wgmma_m64n128k16_rs_tb(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
        "}, {%64, %65, %66, %67}, %68, p, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc));
}

// MN-major SWIZZLE_128B descriptor of a [keys][128 B] tile pair: 64 columns (128 B) per row, 8-row groups 1024 B apart (stride
// byte offset), the next 64 columns `lead` bytes on (leading byte offset)
__device__ __forceinline__ uint64_t gmma_desc_sw128_mn(uint32_t saddr, uint32_t lead) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lead >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit_wait() {
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}

__device__ __forceinline__ void prefill_store(const PrefillParams &p, size_t o, int col, float v0, float v1, float inv) {
    const float a = v0 * inv, c = v1 * inv;
    if (p.out_f32) *reinterpret_cast<float2 *>(p.out_f32 + o * D + col) = make_float2(a, c);
    *reinterpret_cast<uint32_t *>(p.out + o * D + col) = (uint32_t)f32_to_bf16_half_up(a) | ((uint32_t)f32_to_bf16_half_up(c) << 16);
}

// grid (nmb * Hkv); PF_THREADS threads; dynamic smem: Q 32 KB | PF_ST x (K 32 KB | V 32 KB) | barriers, 1024-B aligned
__global__ void __launch_bounds__(PF_THREADS, 1)
    attend_prefill_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                          const __grid_constant__ CUtensorMap map_v, const __grid_constant__ PrefillParams p) {
    extern __shared__ __align__(16) uint8_t pf_raw[];
    uint8_t *sQ = pf_raw + ((1024u - (smem_u32(pf_raw) & 1023u)) & 1023u);
    uint8_t *sKV = sQ + 2 * PF_Q_ATOM;   // stage s: K at sKV + 2s * PF_TILE, V at sKV + (2s + 1) * PF_TILE
    uint64_t *q_full = reinterpret_cast<uint64_t *>(sKV + 2 * PF_ST * PF_TILE), *full = q_full + 1, *empty = full + PF_ST;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mb = p.nmb - 1 - (int)blockIdx.x / p.Hkv, h = (int)blockIdx.x % p.Hkv;   // heaviest m-blocks first
    const int G = p.G, t0 = mb * p.tb, nt = min(p.tb, p.q_len - t0), rows = nt * G;
    const int off = p.kv_len - p.q_len;                                            // query t sees keys [0, off + t]
    const int ntiles = (off + t0 + nt + PF_KT - 1) / PF_KT;

    // rows [tb*G, PF_BM) of the Q tile are never loaded: zero them so that their scores stay finite
    const int pad = PF_BM - p.tb * G;
    for (int c = threadIdx.x; c < pad * 16; c += PF_THREADS) {
        const int a = c / (pad * 8), rem = c - a * pad * 8;
        *reinterpret_cast<uint4 *>(sQ + a * PF_Q_ATOM + (p.tb * G + rem / 8) * 128 + (rem & 7) * 16) = make_uint4(0u, 0u, 0u, 0u);
    }
    fence_proxy_async();   // the zeros before the tensor cores read the tile
    if (threadIdx.x == 0) {
        mbar_init(q_full, 1);
        for (int s = 0; s < PF_ST; ++s) {
            mbar_init(full + s, 1);
            mbar_init(empty + s, 8);   // one arrive per consumer warp
        }
        fence_mbar_init();
        fence_proxy_async();
    }
    __syncthreads();

    if (warp >= 8) {
        // ---------------- TMA producer: hands its registers to the consumers ----------------------------------------------------
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
        if (warp == 8 && lane == 0) {
            expect_tx(q_full, 2u * 128u * (uint32_t)(G * p.tb));
            tma_load_3d(sQ, &map_q, 0, h * G, t0, q_full);
            tma_load_3d(sQ + PF_Q_ATOM, &map_q, 64, h * G, t0, q_full);
            for (int it = 0; it < ntiles; ++it) {
                const int st = it % PF_ST;
                mbar_wait(empty + st, (uint32_t)((it / PF_ST) & 1) ^ 1u);
                expect_tx(full + st, 2 * PF_TILE);
                uint8_t *sk = sKV + (size_t)(2 * st) * PF_TILE, *sv = sk + PF_TILE;
                const int k0 = it * PF_KT;
                tma_load_3d(sk, &map_k, 0, h, k0, full + st);
                tma_load_3d(sk + PF_KV_ATOM, &map_k, 64, h, k0, full + st);
                tma_load_3d(sv, &map_v, 0, h, k0, full + st);
                tma_load_3d(sv + PF_KV_ATOM, &map_v, 64, h, k0, full + st);
            }
        }
        return;
    }
    // ---------------- consumer warpgroups: rows wg*64 + 16*wq + lane/4 (+8) of the m-block -----------------------------------
    asm volatile("setmaxnreg.inc.sync.aligned.u32 240;\n" ::: "memory");
    const int wg = warp >> 2, wq = warp & 3, q4 = lane & 3;
    const int rw = wg * 64 + wq * 16;   // first row of this warp
    int lim[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) lim[i] = off + t0 + (rw + (lane >> 2) + 8 * i) / G;
    const int lim_lo = off + t0 + rw / G;   // the smallest limit of the warp's 16 rows
    const float scale_log2 = rsqrtf((float)D) * LOG2E_F;
    float o[64], s[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) o[j] = 0.f;
    float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_run[2] = {0.f, 0.f};
    const uint32_t qa = smem_u32(sQ) + (uint32_t)(wg * 64 * 128);
    mbar_wait(q_full, 0);

    for (int it = 0; it < ntiles; ++it) {
        const int st = it % PF_ST, k0 = it * PF_KT;
        const uint32_t sk = smem_u32(sKV + (size_t)(2 * st) * PF_TILE), sv = sk + PF_TILE;
        mbar_wait(full + st, (uint32_t)((it / PF_ST) & 1));
        // ---- S = Q . K^T: 64 rows x 128 keys per warpgroup ----------------------------------------------------------------------
        wgmma_fence();
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int k = 0; k < 4; ++k)
                wgmma_m64n128k16_ss(s, gmma_desc_sw128(qa + a * PF_Q_ATOM + k * 32), gmma_desc_sw128(sk + a * PF_KV_ATOM + k * 32),
                                    (a | k) ? 1u : 0u);
        wgmma_commit_wait();
        // ---- causal mask and online softmax (fp32).  Score s[4j + 2i + e] is row i, key k0 + 8j + 2*q4 + e ------------------------
        const bool full_tile = k0 + PF_KT <= p.kv_len && k0 + PF_KT - 1 <= lim_lo;
        float corr[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float mloc = -CUDART_INF_F;
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float &x = s[4 * j + 2 * i + e];
                    const int k = k0 + 8 * j + 2 * q4 + e;
                    x = (full_tile || (k <= lim[i] && k < p.kv_len)) ? x * scale_log2 : -CUDART_INF_F;
                    mloc = fmaxf(mloc, x);
                }
            mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 1));
            mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 2));
            const float m_new = fmaxf(m_run[i], mloc);
            const float m_use = (m_new == -CUDART_INF_F) ? 0.f : m_new;   // a row with no visible key yet: all p = 0
            corr[i] = (m_run[i] == -CUDART_INF_F) ? 0.f : exp2f(m_run[i] - m_new);
            float lsum = 0.f;   // this thread's share; the quad's shares are summed once, after the last tile
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float &x = s[4 * j + 2 * i + e];
                    x = exp2f(x - m_use);
                    lsum += x;
                }
            l_run[i] = l_run[i] * corr[i] + lsum;
            m_run[i] = m_new;
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            o[4 * j] *= corr[0];
            o[4 * j + 1] *= corr[0];
            o[4 * j + 2] *= corr[1];
            o[4 * j + 3] *= corr[1];
        }
        // ---- P as bf16 hi + lo in the A-fragment layout: k16 step ks holds keys 16ks + 2*q4 + {0,1} (regs 0,1) and + 8 (regs 2,3) --
        uint32_t ph[8][4], pl[8][4];
#pragma unroll
        for (int ks = 0; ks < 8; ++ks)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int j = 2 * ks + (r >> 1), i = r & 1;
                const float p0 = s[4 * j + 2 * i], p1 = s[4 * j + 2 * i + 1];
                const uint32_t h0 = f32_to_bf16_rne(p0), h1 = f32_to_bf16_rne(p1);
                const uint32_t l0 = f32_to_bf16_rne(p0 - bf16_bits_to_f32(h0)), l1 = f32_to_bf16_rne(p1 - bf16_bits_to_f32(h1));
                ph[ks][r] = h0 | (h1 << 16);
                pl[ks][r] = l0 | (l1 << 16);
            }
        // ---- O += P . V: V [keys][dims] is the MN-major B operand (next 64 dims one atom on, next 8 keys 1024 B on) ---------------
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            const uint64_t vd = gmma_desc_sw128_mn(sv + ks * 16 * 128, PF_KV_ATOM);
            wgmma_m64n128k16_rs_tb(o, ph[ks], vd);
            wgmma_m64n128k16_rs_tb(o, pl[ks], vd);
        }
        wgmma_commit_wait();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + st);   // this warp's reads of the stage are done
    }

    // ---- epilogue: O / l, row r = t*G + g of the m-block -> (token t0 + t, q-head h*G + g) --------------------------------------
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        float l = l_run[i];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const int r = rw + (lane >> 2) + 8 * i;
        if (r >= rows) continue;
        const int t = r / G, g = r - t * G;
        const size_t orow = (size_t)(t0 + t) * p.Hq + (size_t)h * G + g;
        const float inv = (l > 0.f) ? 1.0f / l : 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) prefill_store(p, orow, 8 * j + 2 * q4, o[4 * j + 2 * i], o[4 * j + 2 * i + 1], inv);
    }
}

// a 3-D bf16 map over an NHD array (n, heads, D): box = 64 dims x box_heads heads x box_rows rows, SWIZZLE_128B, zero fill past n
static int make_map_nhd(CUtensorMap *map, const void *base, int n, int heads, uint32_t box_heads, uint32_t box_rows) {
    PFN_encodeTiled encode;
    int rc = tensor_map_encoder(&encode);
    if (rc) return rc;
    const cuuint64_t dims[3] = {(cuuint64_t)D, (cuuint64_t)heads, (cuuint64_t)n};
    const cuuint64_t strides[2] = {(cuuint64_t)D * 2, (cuuint64_t)heads * D * 2};
    const cuuint32_t box[3] = {64, box_heads, box_rows};
    const cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MPIG_REQUIRE(r == CUDA_SUCCESS, MPIG_ECUDA, "cuTensorMapEncodeTiled failed with %d", (int)r);
    return MPIG_OK;
}

}  // namespace mpig

using namespace mpig;

extern "C" int mpig_prefill_attend(mpig_ctx *ctx, const void *q_bf16, const void *k_bf16, const void *v_bf16, int q_len, int kv_len,
                                   void *out_bf16, float *out_f32, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "mpig_prefill_attend: null context");
    MPIG_REQUIRE(q_bf16 && k_bf16 && v_bf16 && out_bf16, MPIG_EINVAL, "mpig_prefill_attend: null argument");
    MPIG_REQUIRE(q_len >= 1 && kv_len >= q_len, MPIG_EINVAL, "mpig_prefill_attend: need 1 <= q_len <= kv_len (q_len=%d, kv_len=%d)",
                 q_len, kv_len);
    const uintptr_t any = (uintptr_t)q_bf16 | (uintptr_t)k_bf16 | (uintptr_t)v_bf16 | (uintptr_t)out_bf16 | (uintptr_t)out_f32;
    MPIG_REQUIRE((any & 15) == 0, MPIG_EINVAL, "mpig_prefill_attend: q, k, v, out and out_f32 must be 16-byte aligned");
    const int Hq = ctx->cfg.num_attention_heads, Hkv = ctx->cfg.num_key_value_heads, G = ctx->G;
    MPIG_REQUIRE(ctx->cfg.head_dim == D && G >= 1 && G <= 8, MPIG_EUNSUPPORTED,
                 "mpig_prefill_attend: built for head_dim %d and 1 <= Hq / Hkv <= 8 (head_dim %d, G %d)", D, ctx->cfg.head_dim, G);
    PrefillParams p = {};
    p.out = (__nv_bfloat16 *)out_bf16;
    p.out_f32 = out_f32;
    p.q_len = q_len;
    p.kv_len = kv_len;
    p.Hq = Hq;
    p.Hkv = Hkv;
    p.G = G;
    p.tb = PF_BM / G;
    p.nmb = (q_len + p.tb - 1) / p.tb;
    CUtensorMap map_q, map_k, map_v;
    int rc = make_map_nhd(&map_q, q_bf16, q_len, Hq, (uint32_t)G, (uint32_t)p.tb);
    if (!rc) rc = make_map_nhd(&map_k, k_bf16, kv_len, Hkv, 1u, (uint32_t)PF_KT);
    if (!rc) rc = make_map_nhd(&map_v, v_bf16, kv_len, Hkv, 1u, (uint32_t)PF_KT);
    if (rc) return rc;
    MPIG_FUNC_ATTR(attend_prefill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PF_SMEM);
    attend_prefill_kernel<<<(unsigned)p.nmb * (unsigned)Hkv, PF_THREADS, PF_SMEM, as_stream(stream)>>>(map_q, map_k, map_v, p);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}
