// gmma_common.cuh -- the Hopper tensor-core plumbing shared by the wgmma kernels (keyhash.cu, attend_prefill.cu): TMA tensor-map
// loads completed on an mbarrier, the K-major SWIZZLE_128B shared-memory descriptor, and the driver's tensor-map encoder.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace mpig {

__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void tma_load_3d(void *smem_dst, const CUtensorMap *map, int c0, int c1, int c2, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor (8-row x 128-byte atoms, 1024 B apart)
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);   // start address
    d |= (uint64_t)1 << 16;                    // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;          // stride byte offset: next 8-row group
    d |= (uint64_t)1 << 62;                    // SWIZZLE_128B
    return d;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled from the driver the runtime uses (looked up once per translation unit)
static inline int tensor_map_encoder(PFN_encodeTiled *out) {
    static PFN_encodeTiled encode = nullptr;
    if (!encode) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        MPIG_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
        MPIG_REQUIRE(fn && q == cudaDriverEntryPointSuccess, MPIG_ECUDA, "cuTensorMapEncodeTiled entry point not available");
        encode = (PFN_encodeTiled)fn;
    }
    *out = encode;
    return MPIG_OK;
}

}  // namespace mpig
