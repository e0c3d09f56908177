// keyhash.cu -- key-side SimHash on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
// Replaces the prefill-time torch glue of LSHSparseAttnServer.fill (models/attnserver.py:159-168):
//     hash_code = (offload_key[:, chunk] @ hash_func) > 0 ; reshape(-1, K) ; mv with [1,2,4,...] ; transpose ; int16
// i.e. a (Hkv*n x 128) x (128 x K*L) bf16 GEMM (301 GFLOP per layer at P = 98K) whose only output is the SIGN of each
// accumulator, packed little-endian into K-bit codes per table and written in the (Hkv, L, n) int16 layout the table
// build consumes.  The fp32 accumulators never leave the registers: wgmma accumulators -> sign bits -> 2-byte codes, so
// the kernel writes 2*L bytes per key instead of the 4*K*L bytes a plain GEMM would.
//
// One output tile = 128 keys x T tables, T = floor(256 / K), i.e. T*K <= 256 accumulator columns (the wgmma N of 256;
// columns past T*K belong to the next tile's tables and are ignored):
//   TMA      A tile = 128 keys x 128 dims (two 64-column SWIZZLE_128B boxes), B tile = 256 hash vectors x 128 dims from the
//            transposed (K-major) hash_func, completion counted in bytes on an mbarrier
//   wgmma    two consumer warpgroups, 64 keys each: 8 x wgmma.m64n256k16 (fp32 accumulators, 128 registers per thread)
//   epilogue accumulator sign -> per-row 32-bit masks (quad shuffles) -> K-bit codes -> int16 stores
// Rows / tables past the end are zero-filled by TMA (out-of-bounds box) and never stored.
//
// keyhash_pipe_kernel (default) is the persistent, warp-specialised form of the same tile: one CTA per SM walks over key
// tiles; a producer warp keeps two A slots and a ring of B stages filled by TMA (a_full/a_empty, b_full/b_empty), so the
// next tables' B tile is in shared memory while the consumer warpgroups run the MMAs and the sign-pack epilogue of the
// current one.  keyhash_kernel is one tile per CTA.
#include "gmma_common.cuh"

namespace mpig {

constexpr int KH_M = 128;        // keys per tile (two warpgroups of 64)
constexpr int KH_D = 128;        // head_dim
constexpr int KH_N = 256;        // accumulator columns per tile: T = KH_N / K whole tables
constexpr uint32_t KH_A_BYTES = 2u * KH_M * 128u;   // two 64-dim atoms of 128 rows x 128 B
constexpr uint32_t KH_B_BYTES = 2u * KH_N * 128u;   // two 64-dim atoms of 256 rows x 128 B

// D(64 x 256, fp32) (+)= A(64 x 16, smem) * B(16 x 256, smem), both bf16 K-major; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
        "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
        "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127},"
        " %128, %129, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// acc (+)= A rows [64 of the warpgroup] x B (256 columns) over the 128 dims: 2 swizzle atoms x 4 k16 steps
__device__ __forceinline__ void kh_tile_mma(float (&acc)[128], uint32_t a_base, uint32_t b_base) {
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int atom = 0; atom < 2; ++atom)
#pragma unroll
        for (int k = 0; k < 4; ++k)   // 16 bf16 = 32 bytes per k16 step inside the 128-byte swizzle atom
            wgmma_m64n256k16(acc, gmma_desc_sw128(a_base + atom * KH_M * 128 + k * 32),
                             gmma_desc_sw128(b_base + atom * KH_N * 128 + k * 32), (atom | k) ? 1u : 0u);
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}

// Sign-pack epilogue of one warpgroup's 64 x 256 accumulator block.  wgmma layout: thread (warp w, lane l) holds rows
// 16w + l/4 (registers 4i, 4i+1) and 16w + l/4 + 8 (4i+2, 4i+3) at columns 8i + 2(l%4) + {0, 1}.  The four lanes of a quad
// OR their bits into the rows' 32-column masks; lane q of the quad then stores the codes of tables q, q+4, ...
// row0 = first key row of the warpgroup; table t of the tile is table l0 + t (t < t_end).
__device__ __forceinline__ void kh_tile_epilogue(const float (&acc)[128], int16_t *__restrict__ codes, int row0, int rows_total, int n,
                                                 int K, int L, int l0, int t_end, int skip) {
    const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3, q = lane & 3;
    uint32_t m0[8], m1[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {   // bit i of m*[c] = column 32c + i > 0 (attnserver.py:163 .gt(0))
        uint32_t a = 0u, b = 0u;
        if (!(skip & 2)) {
#pragma unroll
            for (int ii = 0; ii < 4; ++ii) {
                const int i = 4 * c + ii, sh = 8 * ii + 2 * q;
                a |= ((uint32_t)(acc[4 * i] > 0.f) << sh) | ((uint32_t)(acc[4 * i + 1] > 0.f) << (sh + 1));
                b |= ((uint32_t)(acc[4 * i + 2] > 0.f) << sh) | ((uint32_t)(acc[4 * i + 3] > 0.f) << (sh + 1));
            }
            a |= __shfl_xor_sync(0xffffffffu, a, 1);
            b |= __shfl_xor_sync(0xffffffffu, b, 1);
            a |= __shfl_xor_sync(0xffffffffu, a, 2);
            b |= __shfl_xor_sync(0xffffffffu, b, 2);
        }
        m0[c] = a;
        m1[c] = b;
    }
    if (skip & 1) return;
    const int r0 = row0 + 16 * wq + (lane >> 2), r1 = r0 + 8;
    const bool ok0 = r0 < rows_total, ok1 = r1 < rows_total;
    const int g0 = ok0 ? r0 / n : 0, j0 = r0 - g0 * n, g1 = ok1 ? r1 / n : 0, j1 = r1 - g1 * n;
    int16_t *dst0 = codes + ((size_t)g0 * L + l0) * n + j0;
    int16_t *dst1 = codes + ((size_t)g1 * L + l0) * n + j1;
    const uint32_t kmask = (1u << K) - 1u;
    for (int t = q; t < t_end; t += 4) {
        const int bit0 = t * K, w = bit0 >> 5, sft = bit0 & 31;   // code = bits [t*K, t*K + K) of the row (attnserver.py:164-165)
        uint32_t lo0 = 0u, hi0 = 0u, lo1 = 0u, hi1 = 0u;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            if (c == w) lo0 = m0[c], lo1 = m1[c];
            if (c == w + 1) hi0 = m0[c], hi1 = m1[c];
        }
        if (ok0) dst0[(size_t)t * n] = (int16_t)((uint32_t)((((uint64_t)hi0 << 32) | lo0) >> sft) & kmask);
        if (ok1) dst1[(size_t)t * n] = (int16_t)((uint32_t)((((uint64_t)hi1 << 32) | lo1) >> sft) & kmask);
    }
}

// grid (n_tiles, m_tiles); 256 threads; dynamic smem: A 32 KB | B 64 KB | barrier, 1024-B aligned
__global__ void __launch_bounds__(256, 1) keyhash_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                                                         int16_t *__restrict__ codes, int rows_total, int n, int K, int L, int T, int skip) {
    extern __shared__ __align__(16) uint8_t kh_smem_raw[];
    // SWIZZLE_128B tiles want 1024-byte aligned shared addresses
    uint8_t *kh_smem = kh_smem_raw + ((1024u - (smem_u32(kh_smem_raw) & 1023u)) & 1023u);
    uint8_t *sA = kh_smem, *sB = kh_smem + KH_A_BYTES;
    uint64_t *bar = reinterpret_cast<uint64_t *>(sB + KH_B_BYTES);
    const int wg = threadIdx.x >> 7;
    const int m0 = blockIdx.y * KH_M, l0 = blockIdx.x * T;

    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
        fence_proxy_async();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        expect_tx(bar, KH_A_BYTES + KH_B_BYTES);
        tma_load_2d(sA, &map_a, 0, m0, bar);                    // dims 0..63
        tma_load_2d(sA + KH_M * 128, &map_a, 64, m0, bar);      // dims 64..127
        tma_load_2d(sB, &map_b, 0, l0 * K, bar);
        tma_load_2d(sB + KH_N * 128, &map_b, 64, l0 * K, bar);
    }
    mbar_wait(bar, 0);
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    if (!(skip & 4)) kh_tile_mma(acc, smem_u32(sA + wg * 64 * 128), smem_u32(sB));
    kh_tile_epilogue(acc, codes, m0 + wg * 64, rows_total, n, K, L, l0, min(T, L - l0), skip);
}

constexpr int KHP_THREADS = 256 + 32;   // two consumer warpgroups + one producer warp
constexpr int KHP_MAX_STAGES = 4;

// persistent grid (<= #SMs CTAs, one per SM); dynamic smem: A slots 2 x 32 KB | B stages nb x 64 KB | barriers
__global__ void __launch_bounds__(KHP_THREADS, 1)
    keyhash_pipe_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, int16_t *__restrict__ codes,
                        int rows_total, int n, int K, int L, int T, int m_tiles, int n_tiles, int nb, int skip) {
    extern __shared__ __align__(16) uint8_t kh_smem_raw[];
    uint8_t *kh_smem = kh_smem_raw + ((1024u - (smem_u32(kh_smem_raw) & 1023u)) & 1023u);
    uint8_t *sA = kh_smem;                                   // [2 slots][2 atoms][128 rows][128 B]
    uint8_t *sB = kh_smem + 2 * (size_t)KH_A_BYTES;          // [nb stages][2 atoms][256 rows][128 B]
    uint64_t *bars = reinterpret_cast<uint64_t *>(sB + (size_t)nb * KH_B_BYTES);
    uint64_t *a_full = bars, *a_empty = bars + 2, *b_full = bars + 4, *b_empty = bars + 4 + KHP_MAX_STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int s = 0; s < 2; ++s) {
            mbar_init(a_full + s, 1);
            mbar_init(a_empty + s, 8);   // one arrive per consumer warp
        }
        for (int s = 0; s < KHP_MAX_STAGES; ++s) {
            mbar_init(b_full + s, 1);
            mbar_init(b_empty + s, 8);
        }
        fence_mbar_init();
        fence_proxy_async();
    }
    __syncthreads();

    if (warp == 8) {
        // ---------------- TMA producer -------------------------------------------------------------------------------
        if (lane == 0) {
            uint32_t it = 0, bcnt = 0;
            for (int mt = blockIdx.x; mt < m_tiles; mt += gridDim.x, ++it) {
                const uint32_t slot = it & 1u, aph = (it >> 1) & 1u;
                mbar_wait(a_empty + slot, aph ^ 1u);
                expect_tx(a_full + slot, KH_A_BYTES);
                uint8_t *da = sA + slot * KH_A_BYTES;
                tma_load_2d(da, &map_a, 0, mt * KH_M, a_full + slot);
                tma_load_2d(da + KH_M * 128, &map_a, 64, mt * KH_M, a_full + slot);
                for (int nt = 0; nt < n_tiles; ++nt, ++bcnt) {
                    const uint32_t st = bcnt % (uint32_t)nb, bph = (bcnt / (uint32_t)nb) & 1u;
                    mbar_wait(b_empty + st, bph ^ 1u);
                    expect_tx(b_full + st, KH_B_BYTES);
                    uint8_t *db = sB + (size_t)st * KH_B_BYTES;
                    tma_load_2d(db, &map_b, 0, nt * T * K, b_full + st);
                    tma_load_2d(db + KH_N * 128, &map_b, 64, nt * T * K, b_full + st);
                }
            }
        }
        return;
    }
    // ---------------- consumer warpgroups 0, 1: 64 key rows each ---------------------------------------------------------
    const int wg = warp >> 2;
    uint32_t it = 0, bcnt = 0;
    float acc[128];
    for (int mt = blockIdx.x; mt < m_tiles; mt += gridDim.x, ++it) {
        const uint32_t slot = it & 1u, aph = (it >> 1) & 1u;
        mbar_wait(a_full + slot, aph);
        const uint32_t a_base = smem_u32(sA + slot * KH_A_BYTES + wg * 64 * 128);
        for (int nt = 0; nt < n_tiles; ++nt, ++bcnt) {
            const uint32_t st = bcnt % (uint32_t)nb, bph = (bcnt / (uint32_t)nb) & 1u;
            mbar_wait(b_full + st, bph);
#pragma unroll
            for (int i = 0; i < 128; ++i) acc[i] = 0.f;
            if (!(skip & 4)) kh_tile_mma(acc, a_base, smem_u32(sB + (size_t)st * KH_B_BYTES));
            // this warp's MMAs have completed: its reads of the B stage are done
            __syncwarp();
            if (lane == 0) mbar_arrive(b_empty + st);
            kh_tile_epilogue(acc, codes, mt * KH_M + wg * 64, rows_total, n, K, L, nt * T, min(T, L - nt * T), skip);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(a_empty + slot);
    }
}

static int make_map_2d(CUtensorMap *map, const void *base, uint64_t rows, uint32_t box_rows) {
    PFN_encodeTiled encode;
    int rc = tensor_map_encoder(&encode);
    if (rc) return rc;
    const cuuint64_t dims[2] = {(cuuint64_t)KH_D, (cuuint64_t)rows};   // innermost first
    const cuuint64_t strides[1] = {(cuuint64_t)KH_D * 2};              // bytes between rows
    const cuuint32_t box[2] = {64, box_rows};                          // 64 bf16 = 128 B = one swizzle atom wide
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MPIG_REQUIRE(r == CUDA_SUCCESS, MPIG_ECUDA, "cuTensorMapEncodeTiled failed with %d", (int)r);
    return MPIG_OK;
}

}  // namespace mpig

using namespace mpig;

extern "C" int mpig_hash_keys(mpig_ctx *ctx, const void *keys_bf16, int n, int16_t *codes_out, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx && codes_out, MPIG_EINVAL, "mpig_hash_keys: null argument");
    MPIG_REQUIRE(n >= 0 && n <= ctx->cfg.max_length, MPIG_EINVAL, "mpig_hash_keys: n=%d exceeds max_length", n);
    if (n == 0) return MPIG_OK;
    MPIG_REQUIRE(ctx->hash_func_set, MPIG_ESTATE, "mpig_hash_keys before mpig_set_hash_func: the projection has not been set");
    MPIG_REQUIRE(keys_bf16, MPIG_EINVAL, "mpig_hash_keys: null keys");
    MPIG_REQUIRE(((uintptr_t)keys_bf16 & 15) == 0, MPIG_EINVAL, "mpig_hash_keys: keys must be 16-byte aligned");
    const int K = ctx->cfg.K, L = ctx->cfg.L, Hkv = ctx->cfg.num_key_value_heads;
    const int T = KH_N / K;   // whole tables per tile
    const long rows = (long)Hkv * n;
    CUtensorMap map_a, map_b;
    int rc = make_map_2d(&map_a, keys_bf16, (uint64_t)rows, KH_M);
    if (rc) return rc;
    rc = make_map_2d(&map_b, ctx->hash_func_t, (uint64_t)K * L, (uint32_t)KH_N);
    if (rc) return rc;
    const int m_tiles = (int)((rows + KH_M - 1) / KH_M);
    const int n_tiles = (L + T - 1) / T;
    if (ctx->keyhash_impl == 1) {
        // B stages: as many as fit beside the two A slots (2 on sm_90a)
        const size_t fixed = 1024 + 128;
        int nb = (int)((227 * 1024 - 2 * (size_t)KH_A_BYTES - fixed) / KH_B_BYTES);
        if (nb > KHP_MAX_STAGES) nb = KHP_MAX_STAGES;
        const size_t smem = 2 * (size_t)KH_A_BYTES + (size_t)nb * KH_B_BYTES + fixed;
        MPIG_FUNC_ATTR(keyhash_pipe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        const int grid = m_tiles < ctx->num_sms ? m_tiles : ctx->num_sms;
        keyhash_pipe_kernel<<<grid, KHP_THREADS, smem, as_stream(stream)>>>(map_a, map_b, codes_out, (int)rows, n, K, L, T, m_tiles,
                                                                          n_tiles, nb, ctx->keyhash_skip);
        MPIG_LAUNCH_CHECK(ctx);
        return MPIG_OK;
    }
    const size_t smem = (size_t)KH_A_BYTES + KH_B_BYTES + 64 + 1024;
    MPIG_FUNC_ATTR(keyhash_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    keyhash_kernel<<<dim3(n_tiles, m_tiles), 256, smem, as_stream(stream)>>>(map_a, map_b, codes_out, (int)rows, n, K, L, T,
                                                                             ctx->keyhash_skip);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}
