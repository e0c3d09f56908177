// Micro-benchmark: latency of ONE dependent global load per warp when every warp of a full grid issues it at once.
#include <cuda_runtime.h>
#include <cstdio>
#include <vector>
#include <algorithm>
extern __shared__ int dsm[];
__global__ void k(const int* __restrict__ buf, size_t stride_elems, int per_head, long long* out, int mode) {
    if (threadIdx.x == 0) dsm[0] = 1;
    __syncthreads();
    int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    int head = warp / per_head, part = warp % per_head;
    long long t0;
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(t0));
    const int* p = buf + (size_t)head * stride_elems + (size_t)part * 32 + lane + (int)(t0 & 0);  // address depends on t0
    int v;
    if (mode == 0) asm volatile("ld.global.nc.b32 %0, [%1];" : "=r"(v) : "l"(p));
    else if (mode == 1) asm volatile("ld.global.b32 %0, [%1];" : "=r"(v) : "l"(p));
    else if (mode == 2) asm volatile("ld.global.cg.b32 %0, [%1];" : "=r"(v) : "l"(p));
    else asm volatile("ld.volatile.global.b32 %0, [%1];" : "=r"(v) : "l"(p));
    long long t1;
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(t1) : "r"(v));
    if (lane == 0) out[warp] = t1 - t0;
}
int main() {
    int warps = 132 * 12;   // 12 warps on each of an H100 SXM's 132 SMs
    size_t stride = 98304;
    int heads = 32, per_head = (warps + heads - 1) / heads;
    std::vector<int*> bufs;
    for (int i = 0; i < 40; ++i) { int* b; cudaMalloc(&b, heads * stride * 4); cudaMemset(b, 0, heads * stride * 4); bufs.push_back(b); }
    long long* out; cudaMalloc(&out, warps * 8);
    std::vector<long long> h(warps);
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    const char* names[4] = {"ld.global.nc", "ld.global", "ld.global.cg", "ld.volatile"};
    for (int smem_kb : {1, 211}) {
        for (int mode = 0; mode < 4; ++mode) {
            for (int rep = 0; rep < 2; ++rep) {
                int* b = bufs[(mode * 9 + smem_kb) % bufs.size()];   // rep 0: cold buffer, rep 1: same lines again (L2 resident)
                k<<<132, 384, smem_kb * 1024>>>(b, stride, per_head, out, mode);
                cudaDeviceSynchronize();
                cudaMemcpy(h.data(), out, warps * 8, cudaMemcpyDeviceToHost);
                std::sort(h.begin(), h.end());
                printf("smem %3d KB %-14s %s: cycles p10 %5lld  p50 %5lld  p90 %5lld  max %5lld\n", smem_kb, names[mode], rep ? "L2-warm" : "cold   ",
                       h[warps / 10], h[warps / 2], h[warps * 9 / 10], h[warps - 1]);
            }
        }
    }
    return 0;
}
