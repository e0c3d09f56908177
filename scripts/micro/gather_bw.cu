// Micro-benchmark: what the HBM system delivers for the fused kernel's row fetch and nothing else.
// 128 CTAs (one per SM, 1024 threads, ~200 KB of row buffers) each fetch R random 512-byte records of their own key range with
// one cp.async.bulk per record -- the access pattern of fused_decode_kernel's attend phase at C2 (32 heads x 4 key ranges of
// 24.5K records, ~400 sampled records per CTA, ascending within the CTA) -- wait for all of them, and exit.  Buffers rotate so
// that every launch reads cold lines.  Reported: launch time (CUDA events), in-kernel time from the first request to the last
// arrival, and the fit  t(R) = t0 + bytes / BW  over R.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o gather_bw gather_bw.cu && ./gather_bw
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

constexpr int REC = 512, ROWS_PER_WARP = 16, MAXW = 26;   // 26 row buffers of 16 records, as the fused kernel has at C2

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__global__ void __launch_bounds__(1024, 1) gather_kernel(const uint8_t *__restrict__ kv, const int *__restrict__ idx, int R, size_t rows_per_head,
                                                          int ctas_per_head, long long *__restrict__ t_out, float *__restrict__ sink) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t bars[32];
    __shared__ long long t_first, t_last;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int head = blockIdx.x / ctas_per_head;
    if (lane == 0 && warp < MAXW) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bars[warp])));
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    if (threadIdx.x == 0) { t_first = 0x7fffffffffffffffll; t_last = 0; }
    __syncthreads();
    long long t0;
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(t0));
    float acc = 0.f;
    uint32_t phase = 0;
    if (warp < MAXW) {
        uint8_t *buf = smem + (size_t)warp * ROWS_PER_WARP * REC;
        for (int r0 = warp * ROWS_PER_WARP; r0 < R; r0 += MAXW * ROWS_PER_WARP) {
            const int n = min(ROWS_PER_WARP, R - r0);
            if (lane == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bars[warp])), "r"(n * REC) : "memory");
            __syncwarp();
            if (lane < n) {
                const uint8_t *src = kv + ((size_t)head * rows_per_head + idx[(size_t)blockIdx.x * R + r0 + lane]) * REC;
                asm volatile("cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(buf + lane * REC)),
                             "l"(src), "r"(REC), "r"(smem_u32(&bars[warp]))
                             : "memory");
            }
            uint32_t done = 0;
            while (!done)
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(smem_u32(&bars[warp])), "r"(phase) : "memory");
            phase ^= 1;
            acc += reinterpret_cast<const float *>(buf)[lane * 7];   // touch the data
            __syncwarp();
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        }
    }
    long long t1;
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(t1));
    if (lane == 0 && warp < MAXW) { atomicMin(&t_first, t0); atomicMax(&t_last, t1); }
    __syncthreads();
    if (threadIdx.x == 0) t_out[blockIdx.x] = t_last - t_first;
    if (acc == 123.456f) sink[0] = acc;
}

int main() {
    const int heads = 32, cph = 4, ctas = heads * cph, kvh = 8;
    const size_t rows_per_head = 98304, seg = rows_per_head / cph;
    const size_t bytes = kvh * rows_per_head * REC;   // one layer's records (402 MB): > the 50 MB L2
    const int NBUF = 6;
    std::vector<uint8_t *> bufs(NBUF);
    for (auto &b : bufs) { cudaMalloc(&b, bytes); cudaMemset(b, 1, bytes); }
    long long *t_out; cudaMalloc(&t_out, ctas * 8);
    float *sink; cudaMalloc(&sink, 4);
    int clk_khz = 0; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    cudaFuncSetAttribute(gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MAXW * ROWS_PER_WARP * REC);
    std::mt19937 rng(1);
    printf("random 512-byte record gather, %d CTAs x 1024 threads, %d row buffers of %d records per CTA, SM clock %d MHz\n", ctas, MAXW, ROWS_PER_WARP, clk_khz / 1000);
    printf("%8s %10s %12s %14s %14s\n", "rows/CTA", "MB/launch", "launch us", "in-kernel us", "GB/s (launch)");
    std::vector<double> xs, ys;
    for (int R : {16, 104, 208, 416, 832, 1664}) {
        std::vector<int> h((size_t)ctas * R);
        for (int c = 0; c < ctas; ++c) {
            std::vector<int> v(R);
            for (auto &x : v) x = (int)((c % cph) * seg + rng() % seg);
            std::sort(v.begin(), v.end());
            std::copy(v.begin(), v.end(), h.begin() + (size_t)c * R);
        }
        int *idx; cudaMalloc(&idx, h.size() * 4);
        cudaMemcpy(idx, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        // the q-heads of a GQA group read the same kv-head's records: head -> kv-head = head / 4
        auto launch = [&](int b) { gather_kernel<<<ctas, 1024, MAXW * ROWS_PER_WARP * REC>>>(bufs[b % NBUF] - 0, idx, R, rows_per_head, cph * 4, t_out, sink); };
        for (int w = 0; w < 3; ++w) launch(w);
        cudaDeviceSynchronize();
        const int reps = 24;
        cudaEventRecord(e0);
        for (int i = 0; i < reps; ++i) launch(i);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        std::vector<long long> t(ctas);
        cudaMemcpy(t.data(), t_out, ctas * 8, cudaMemcpyDeviceToHost);
        std::sort(t.begin(), t.end());
        const double us = ms * 1e3 / reps, mb = (double)ctas * R * REC / 1e6, inker = t[ctas / 2] / (clk_khz / 1e3);
        printf("%8d %10.2f %12.2f %14.2f %14.0f\n", R, mb, us, inker, mb * 1e6 / us / 1e3);
        xs.push_back(mb); ys.push_back(us);
        cudaFree(idx);
    }
    // least-squares fit over the four largest sizes: us = t0 + MB / BW
    double sx = 0, sy = 0, sxx = 0, sxy = 0; int n = 0;
    for (size_t i = 2; i < xs.size(); ++i) { sx += xs[i]; sy += ys[i]; sxx += xs[i] * xs[i]; sxy += xs[i] * ys[i]; ++n; }
    const double slope = (n * sxy - sx * sy) / (n * sxx - sx * sx), t0 = (sy - slope * sx) / n;
    printf("fit over the four largest: t = %.2f us + bytes / %.0f GB/s\n", t0, 1e3 / slope);
    return 0;
}
