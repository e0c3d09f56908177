// probe_common.cuh -- device helpers shared by the probe kernel (tables.cu) and the fused decode kernel (fused.cu)
#pragma once
#include "common.cuh"

namespace mpig {

// ---------------------------------------------------------------------------------------------
// block-wide exclusive scan of one int per thread (blockDim.x multiple of 32, <= 1024)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int block_exclusive_scan(int v, int *warp_sums /* >= 33 ints */, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int w = (lane < nwarps) ? warp_sums[lane] : 0;
        int winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, winc, o);
            if (lane >= o) winc += t;
        }
        if (lane < nwarps) warp_sums[lane] = winc - w;  // exclusive warp offsets
        if (lane == 31) warp_sums[32] = winc;           // grand total
    }
    __syncthreads();
    int res = warp_sums[warp] + inc - v;
    *total = warp_sums[32];
    __syncthreads();  // warp_sums may be reused by the caller
    return res;
}

__device__ __forceinline__ unsigned cluster_ctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ unsigned cluster_nctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_barrier() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// Split cluster barrier.  A CTA may only store into a peer's shared memory once that peer has started executing (the
// programming model's rule; compute-sanitizer racecheck flags the violation): every thread ARRIVES at kernel entry and WAITS
// right before the kernel's first remote store -- by then every CTA of the cluster has long arrived, so the wait is free.
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void st_shared_cluster_u32(const void *local_smem_addr, unsigned target_rank, uint32_t v) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local_smem_addr)), "r"(target_rank));
    asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(remote), "r"(v) : "memory");
}

// block-wide exclusive scan with ONE barrier: warp scans -> per-warp totals in shared memory -> every warp scans the totals
// itself.  `wtot` needs >= 32 ints and must not be reused before the caller's next barrier.
__device__ __forceinline__ int block_exclusive_scan_1bar(int v, int *wtot, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) wtot[warp] = inc;
    __syncthreads();
    const int w = (lane < nwarps) ? wtot[lane] : 0;
    int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, winc, o);
        if (lane >= o) winc += t;
    }
    *total = __shfl_sync(0xffffffffu, winc, 31);
    return __shfl_sync(0xffffffffu, winc - w, warp) + inc - v;
}

// 128-bit store into the shared memory of CTA `target_rank` of the cluster
__device__ __forceinline__ void st_shared_cluster_f4(const void *local_smem_addr, unsigned target_rank, float4 v) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local_smem_addr)), "r"(target_rank));
    asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(remote), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Shared spill mode (DESIGN.md section 3.12): drop from the tags of this CTA's key range [lo_key, lo_key + Mc) the private keys of
// the slot that request b does not see.  Keys >= plo (the slot's prompt key count) are private; private key k is seen by b iff bit
// b of vis_slot[k - plo] is set.  Every tag of such a key that is not EMPTY (one collision or SEL) becomes EMPTY, so the selection,
// nnz, the index list and the collision bitmaps all see the request's own context.  vis is written by kernels (spill, fork, bind):
// call it after griddepcontrol.wait.  Ends with a barrier.
template <typename TagT>
__device__ __noinline__ void filter_private(TagT *tag, const uint32_t *vis_slot, int plo, int lo_key, int Mc, int b) {
    constexpr TagT EMPTY = (TagT)((TagT)(~(TagT)0) - 1);
    for (int i = max(plo - lo_key, 0) + (int)threadIdx.x; i < Mc; i += (int)blockDim.x)
        if (tag[i] != EMPTY && !((__ldcg(vis_slot + (lo_key + i - plo)) >> b) & 1u)) tag[i] = EMPTY;
    __syncthreads();
}

// cluster geometry of a probe: S key segments (padded to a power of two Sp) x r CTAs per segment, C = Sp*r <= 8 CTAs per
// q-head, each owning Mc keys (one tag each) of one segment
struct ProbeGeom {
    int Sp, r, C, Mc;
};
ProbeGeom probe_geometry(const mpig_ctx *ctx);   // tables.cu

}  // namespace mpig
