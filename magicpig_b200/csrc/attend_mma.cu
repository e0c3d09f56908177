// attend_mma.cu -- stage 3 as a stand-alone kernel: importance-weighted gather attention over a given index list
// (+ the window rows when the caller passes them), i.e. SparseAttentionServer::attention_wrapper.
//
// Replaces library/sparse_attention/sparse_attention.cc:
//   attention_wrapper / attention(_bf16) :629-745, :867-986
//     qk_kernel(_bf16_impl)  :38-103,  transform_kernel :164-184,
//     softmax_kernel         :186-240, wv_kernel        :321-347     -> attend_mma_kernel (one pass, fused)
// mpig_decode runs the same tile math inside the fused per-layer kernel (fused.cu); this kernel serves
// mpig_attention_wrapper and the three-launch decode variant (option "decode_impl" = 0).
//
// Data movement.  Each warp owns 32 record slots in shared memory.  Lane i of the warp resolves row i of the tile (index ->
// record address) and issues ONE 512-byte `cp.async.bulk` (TMA engine, SASS UBLKCP) from HBM into slot i; completion is
// counted in bytes on the warp's mbarrier.  12 warps per SM keep 196 KB in flight per SM.
// Tile math (32 rows per warp):
//   S = K_tile (32 x 128, bf16, smem) . q (128, bf16)         2 m-tiles x 8 k-steps of mma.m16n8k16, A = K rows via
//                                                              ldmatrix.x4, B = q in column 0 (fp32 accumulate, exact products)
//   lane r owns row r: cos -> theta -> p -> w -> z = s/sqrt(d) - ln(w + 1e-4)   (transform_kernel); the two integer powers
//                                                              by repeated squaring in fp64, rounded to fp32 once
//   online softmax (running max / sum, base-2 exponentials)
//   o += P (1 x 32) . V_tile (32 x 128, bf16, smem)            on the FP32 pipe: with one query row per warp an m16n8k16 would spend
//                                                              14 of its 16 A rows on zeros, and legacy mma.sync issues at ~1 per 32
//                                                              cycles per SM sub-partition on this part (measured: 1.9 us of an 18 us
//                                                              kernel as HMMA vs ~0.5 us as FFMA)
// The shared-memory slot stride is 528 B (512 + 16): 8 consecutive rows then start in 8 different 16-byte bank
// groups, which is what makes the ldmatrix pattern conflict-free.
#include "attend_common.cuh"

namespace mpig {

// Stage timestamps for scripts/attend_timeline.py.  Kept in REGISTERS (per-SM 32-bit cycle counter) and written out once
// at the very end of the kernel, so that the instrumentation adds no memory traffic to the path it measures; compiled
// only into the DBG instantiation of the kernel.
__device__ __forceinline__ uint32_t clk32() {
    uint32_t t;
    asm volatile("mov.u32 %0, %%clock;" : "=r"(t));
    return t;
}
__device__ __forceinline__ uint32_t clk32_after(int dep) {
    uint32_t t;
    asm volatile("mov.u32 %0, %%clock;" : "=r"(t) : "r"(dep));
    return t;
}
#define DBG_STAMP(k)                  \
    do {                              \
        if (DBG) dbg_t[(k)] = clk32(); \
    } while (0)
#define DBG_STAMP_DEP(k, dep)                          \
    do {                                               \
        if (DBG) dbg_t[(k)] = clk32_after((int)(dep)); \
    } while (0)
#define DBG_FLUSH()                                                                                      \
    do {                                                                                                 \
        if (DBG && p.dbg && lane == 0) {                                                                 \
            _Pragma("unroll") for (int k_ = 0; k_ < 16; ++k_) p.dbg[(size_t)u_dbg * 16 + k_] = dbg_t[k_]; \
        }                                                                                                \
    } while (0)

// Work decomposition (head-aligned stream-K).  Head h owns T_h = W_b + nnz_h rows.  With nw warps in the grid,
//   Rp  = max(32, ceil(total / (nw - H)))            rows a warp should take
//   w_h = max(1, floor(T_h / Rp))                    warps ("parts") of head h;  sum_h w_h <= nw
//   part k of head h = rows [k*c_h, (k+1)*c_h),  c_h = ceil(T_h / w_h)
// so every warp works on exactly ONE head (a single latency chain per warp: resolve rows -> fetch -> math ->
// publish), parts differ by at most one row inside a head, and heads with more sampled keys simply get more
// warps.  Parts are numbered consecutively over heads ("items"); item i is processed by warp i of the grid, so
// the parts of one head sit in neighbouring warps / CTAs and are combined in two levels, each by the last
// contributor to arrive (acq_rel ticket counters, no barrier, no second kernel):
//   level 1  parts inside one CTA      -> shared-memory slots + shared-memory ticket
//   level 2  CTAs that share the head  -> global scratch slots (2 per CTA: head entering / head leaving) + ticket
// smem: ring [warps][32][528] | bars [warps rounded up to even] u64 | s_part [warps][132] f32 | s_own [warps][132] f32
//       | s_cnt [warps] | s_wlen [B] | s_prefix [H+1] | s_wpre [H+1]
template <bool USE_TMA, bool DBG>
__global__ void __launch_bounds__(384, 1) attend_mma_kernel(const __grid_constant__ AttendParams gp) {
    extern __shared__ __align__(128) uint8_t smem[];
    // Kernel parameters live in the constant bank; every use is a separate LDC and the first touch of each
    // constant line after a launch is a long miss, which serialised into several microseconds on each warp's critical
    // path.  They are staged ONCE into shared memory (one parallel burst of LDCs) and read from there afterwards.
    __shared__ AttendParams p_smem;
    {
        constexpr int NW32 = (int)(sizeof(AttendParams) / 4);
        for (int i = threadIdx.x; i < NW32; i += blockDim.x)
            reinterpret_cast<uint32_t *>(&p_smem)[i] = reinterpret_cast<const uint32_t *>(&gp)[i];
    }
    __syncthreads();
    const AttendParams &p = p_smem;
    const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t *slots = smem + (size_t)warp * TILE * SLOT;
    uint8_t *sp = smem + (size_t)warps * TILE * SLOT;
    uint64_t *bar = reinterpret_cast<uint64_t *>(sp) + warp;
    sp += (size_t)((warps + 1) & ~1) * sizeof(uint64_t);   // padded to 16 bytes: the state slots below are read / written as float4
    float *s_part = reinterpret_cast<float *>(sp);
    sp += (size_t)warps * PART_FLOATS * sizeof(float);
    float *s_own = reinterpret_cast<float *>(sp) + (size_t)warp * PART_FLOATS;
    sp += (size_t)warps * PART_FLOATS * sizeof(float);
    int *s_cnt = reinterpret_cast<int *>(sp);
    sp += (size_t)warps * sizeof(int);
    int *s_wlen = reinterpret_cast<int *>(sp);
    const int Bn = p.H / p.Hq;
    int *s_prefix = s_wlen + Bn;      // rows before head h
    int *s_wpre = s_prefix + p.H + 1;  // items (warp parts) before head h

    const int u_dbg = blockIdx.x * warps + warp;
    uint32_t dbg_t[16];
#pragma unroll
    for (int k_ = 0; k_ < 16; ++k_) dbg_t[k_] = 0u;
    DBG_STAMP(0);
    if (lane == 0) {
        mbar_init(bar, 1);
        fence_proxy_async();  // init visible to the async proxy (a cluster-scope mbarrier_init fence costs an L1 invalidate: ~4.7 us measured)
    }
    if (threadIdx.x < warps) s_cnt[threadIdx.x] = 0;
    // everything above is independent of the producer kernel (probe) -> overlaps its tail under PDL
    pdl_wait();

    const int nw = gridDim.x * warps;
    if (warp == 0) {
        for (int b = lane; b < Bn; b += 32) s_wlen[b] = p.win ? min(max(p.win_len[b], 0), p.Wcap) : 0;
        __syncwarp();
        int run = 0;
        for (int h0 = 0; h0 < p.H; h0 += 32) {
            const int h = h0 + lane;
            int t = 0;
            if (h < p.H) t = s_wlen[h / p.Hq] + (p.nnz ? min(max(p.nnz[h], 0), p.M) : 0);
            int inc = t;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int v = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += v;
            }
            if (h < p.H) s_prefix[h] = run + inc - t;
            run += __shfl_sync(0xffffffffu, inc, 31);
        }
        const int total = run;
        if (lane == 0) s_prefix[p.H] = total;
        // parts per head
        const int Rp = (nw > p.H) ? max(TILE, (total + (nw - p.H) - 1) / (nw - p.H)) : 0x3fffffff;
        __syncwarp();
        run = 0;
        for (int h0 = 0; h0 < p.H; h0 += 32) {
            const int h = h0 + lane;
            int w = 0;
            if (h < p.H) {
                const int t = s_prefix[h + 1] - s_prefix[h];
                w = (t > 0) ? max(1, t / Rp) : 0;
            }
            int inc = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int v = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += v;
            }
            if (h < p.H) s_wpre[h] = run + inc - w;
            run += __shfl_sync(0xffffffffu, inc, 31);
        }
        if (lane == 0) s_wpre[p.H] = run;
    }
    __syncthreads();
    pdl_launch_dependents();
    DBG_STAMP(1);

    const int u = blockIdx.x * warps + warp;
    const int n_items = s_wpre[p.H];
    const int cta_w0 = blockIdx.x * warps;  // first global warp id of this CTA

    // heads with no rows at all still owe an output (SURVEY 7.3 #7: zeros, LSE = -inf)
    for (int h = u; h < p.H; h += nw) {
        if (s_prefix[h + 1] == s_prefix[h]) {
            const float z4[4] = {0.f, 0.f, 0.f, 0.f};
            finalize_head(p, h, -CUDART_INF_F, 0.f, z4, lane);
        }
    }

    const float inv_sqrt_dim = rsqrtf((float)D);
    const float Lf = (float)p.L;
    const int grp = lane >> 2, tig = lane & 3;
    const uint32_t slots_s = smem_u32(slots);
    // ldmatrix lane addresses (bytes inside the tile): A operand rows of K, B operand rows of V (transposed load)
    const uint32_t a_lane_off = (uint32_t)(((lane & 7) + ((lane >> 3) & 1) * 8) * SLOT + (lane >> 4) * 16);
    const uint32_t v_lane_off = (uint32_t)(((lane & 7) + ((lane >> 3) & 1) * 8) * SLOT + D * 2 + (lane >> 4) * 16);
    uint32_t phase = 0;

    for (int item = u; item < n_items; item += nw) {
        // which head / which part
        int ch;
        {
            int a = 0, b = p.H;
            while (b - a > 1) {
                const int mid = (a + b) >> 1;
                if (s_wpre[mid] <= item) a = mid; else b = mid;
            }
            ch = a;
            while (s_wpre[ch + 1] <= item) ++ch;  // heads without parts share the same prefix value
        }
        const int T = s_prefix[ch + 1] - s_prefix[ch];
        const int w_h = s_wpre[ch + 1] - s_wpre[ch];
        const int part = item - s_wpre[ch];
        const int c_h = (T + w_h - 1) / w_h;
        const int r_lo = part * c_h, r_hi = min(r_lo + c_h, T);  // rows of this part inside the head's list
        const int g = ch / p.G;
        const int sg = p.slot_of ? p.slot_of[ch / p.Hq] * (p.Hq / p.G) + (ch % p.Hq) / p.G : g;   // slot group of the sampled rows
        const int wlen = s_wlen[ch / p.Hq];

        DBG_STAMP_DEP(12, wlen);  // head / part resolved
        // q row (256 B) and |q|: ONE coalesced load per warp, issued after the first tile's row copies (below) so that
        // the row-index load is not queued behind it; the mma B fragments are formed from it by shuffles.
        uint32_t qb[8][2];
        float qn = 1.f;
        bool have_q = false;

        float m_run = -CUDART_INF_F, l_run = 0.f;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};  // lane owns output dims 4*lane .. 4*lane+3

        DBG_STAMP_DEP(14, r_hi);  // part bounds known, accumulators cleared
        for (int cr = r_lo; cr < r_hi; cr += TILE) {
            const int nrows = min(TILE, r_hi - cr);
            // ---- fetch: lane r resolves row r; the record travels either as one 512-byte bulk copy issued by that
            //      lane (TMA engine) or, row by row, as 32 x 16-byte cp.async from the whole warp (LSU path) --------
            float meta = -1.0f;
            const bool do_fetch = !(p.skip & 1), do_math = !(p.skip & 2);
            if (USE_TMA && do_fetch) {
                if (lane == 0) mbar_arrive_expect_tx(bar, (uint32_t)nrows * REC);
                __syncwarp();
            }
            DBG_STAMP(13);  // barrier armed
            const uint8_t *src = nullptr;
            if (lane < nrows) {
                const int j = cr + lane;  // position in the head's row list
                int idx = -1;
                if (j < wlen) {
                    src = p.win + ((size_t)g * p.Wcap + j) * REC;
                } else {
                    const int32_t *ip = p.ind + (size_t)ch * p.M + (j - wlen);
                    DBG_STAMP_DEP(15, (int)(size_t)ip);  // address ready
                    idx = __ldg(ip);
                    idx = min(max(idx, 0), p.M - 1);
                    src = p.kv + ((size_t)sg * p.M + idx) * REC;
                }
                if (USE_TMA && do_fetch) bulk_g2s(slots + (size_t)lane * SLOT, src, REC, bar);
                if (idx >= 0) meta = __ldg(p.kn + (size_t)sg * p.M + idx);  // consumed in phase B: overlaps the row fetch
            }
            if (!USE_TMA && do_fetch) {
                const unsigned long long sp64 = (unsigned long long)src;
                for (int r = 0; r < nrows; ++r) {
                    const unsigned long long a = __shfl_sync(0xffffffffu, sp64, r);
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(slots_s + (uint32_t)(r * SLOT + lane * 16)),
                                 "l"(a + (unsigned long long)lane * 16)
                                 : "memory");
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
            }
            DBG_STAMP(2);  // row copies issued
            if (!have_q) {
                const uint32_t *q32 = reinterpret_cast<const uint32_t *>(p.q + (size_t)ch * D);
                const uint32_t qw0 = __ldg(q32 + lane), qw1 = __ldg(q32 + 32 + lane);  // words lane and lane+32
                const float qn0 = __ldg(p.qnorm + ch);
#pragma unroll
                for (int ks = 0; ks < 8; ++ks) {
                    // B fragment of column 0: words ks*8 + tig and ks*8 + 4 + tig of the q row (lanes with grp == 0)
                    const uint32_t src = (ks < 4) ? qw0 : qw1;
                    const uint32_t b0 = __shfl_sync(0xffffffffu, src, (ks & 3) * 8 + tig);
                    const uint32_t b1 = __shfl_sync(0xffffffffu, src, (ks & 3) * 8 + 4 + tig);
                    qb[ks][0] = (grp == 0) ? b0 : 0u;
                    qb[ks][1] = (grp == 0) ? b1 : 0u;
                }
                qn = qn0;
                have_q = true;
            }
            if (!do_fetch) {
                __syncwarp();
            } else if (USE_TMA) {
                __syncwarp();  // zero fill visible to the whole warp before ldmatrix
                mbar_wait(bar, phase);
                phase ^= 1;
            } else {
                asm volatile("cp.async.wait_group 0;" ::: "memory");
                __syncwarp();
            }
            DBG_STAMP(3);  // tile landed

            if (do_math) {
                // ---- A: scores on the tensor cores ---------------------------------------------------------------
                float sc[2][2];
    #pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
    #pragma unroll
                    if (!(p.skip & 8)) {
#pragma unroll
                        for (int ks = 0; ks < 8; ++ks) {
                            uint32_t a[4];
                            ldsm_x4(a, slots_s + (uint32_t)(mt * 16 * SLOT + ks * 32) + a_lane_off);
                            mma_16816(c0, c1, c2, c3, a, qb[ks][0], qb[ks][1]);
                        }
                    }
                    sc[mt][0] = c0;  // row mt*16 + grp      (column 0 lives in lanes with tig == 0)
                    sc[mt][1] = c2;  // row mt*16 + 8 + grp
                }
                float s_mine = 0.f;
    #pragma unroll
                for (int mt = 0; mt < 2; ++mt)
    #pragma unroll
                    for (int hf = 0; hf < 2; ++hf) {
                        const float got = __shfl_sync(0xffffffffu, sc[mt][hf], 4 * (lane & 7));
                        if ((lane >> 3) == mt * 2 + hf) s_mine = got;
                    }
                DBG_STAMP(4);

                // ---- B: LSH-probability re-weighting (transform_kernel :173-183) --------------------------------
                float z = -CUDART_INF_F;
                if (lane < nrows) {
                    z = s_mine * inv_sqrt_dim;
                    if (meta >= 0.f && !(p.skip & 16)) {
                        float cs = s_mine / (qn * meta);
                        cs = fminf(fmaxf(cs, -1.0f), 1.0f);  // the reference would produce NaN past +-1
                        const float theta = fast_acosf(cs);
                        const float proba = 1.0f - theta * 0.318309886183790672f;
                        const float w = sample_weight(proba, p.K, p.L, Lf);
                        z -= __logf(w + 1e-4f);
                    }
                }
                DBG_STAMP(5);

                // ---- C: online softmax ---------------------------------------------------------------------------
                const float m_new = fmaxf(m_run, warp_max(z));
                const float corr = (m_run == -CUDART_INF_F) ? 0.f : exp2f((m_run - m_new) * LOG2E_F);
                const float pj = (lane < nrows) ? exp2f((z - m_new) * LOG2E_F) : 0.f;
                l_run = l_run * corr + warp_sum(pj);
                m_run = m_new;
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[i] *= corr;
                DBG_STAMP(6);

                // ---- D: o += p_r * V_r on the FP32 pipe: p_r broadcast by shuffle, lane owns 4 dims, 4 rows in flight ----
                if (!(p.skip & 32)) {
                    const uint8_t *vbase = slots + D * 2 + lane * 8;
                    int r = 0;
                    for (; r + 4 <= nrows; r += 4) {
                        uint2 vv[4];
                        float pv[4];
#pragma unroll
                        for (int uu = 0; uu < 4; ++uu) {
                            vv[uu] = *reinterpret_cast<const uint2 *>(vbase + (size_t)(r + uu) * SLOT);
                            pv[uu] = __shfl_sync(0xffffffffu, pj, r + uu);
                        }
#pragma unroll
                        for (int uu = 0; uu < 4; ++uu) {
                            acc[0] = fmaf(pv[uu], bf16lo(vv[uu].x), acc[0]);
                            acc[1] = fmaf(pv[uu], bf16hi(vv[uu].x), acc[1]);
                            acc[2] = fmaf(pv[uu], bf16lo(vv[uu].y), acc[2]);
                            acc[3] = fmaf(pv[uu], bf16hi(vv[uu].y), acc[3]);
                        }
                    }
                    for (; r < nrows; ++r) {
                        const uint2 v = *reinterpret_cast<const uint2 *>(vbase + (size_t)r * SLOT);
                        const float pv = __shfl_sync(0xffffffffu, pj, r);
                        acc[0] = fmaf(pv, bf16lo(v.x), acc[0]);
                        acc[1] = fmaf(pv, bf16hi(v.x), acc[1]);
                        acc[2] = fmaf(pv, bf16lo(v.y), acc[2]);
                        acc[3] = fmaf(pv, bf16hi(v.y), acc[3]);
                    }
                }
            } else {
                m_run = 0.f;
                l_run = 1.f + meta;
            }
            __syncwarp();
            fence_proxy_async();  // this tile's generic-proxy reads precede the next tile's async-proxy writes
            DBG_STAMP(7);
        }

        // ---- this part is done ------------------------------------------------------------------------------------
        float A[4] = {acc[0], acc[1], acc[2], acc[3]};
        float M_ = m_run, L_ = l_run;
        DBG_STAMP(8);

        if (w_h == 1 || (p.skip & 4)) {
            finalize_head(p, ch, M_, L_, A, lane);
            DBG_FLUSH();
            continue;
        }
        // the head's parts are items [i0, i1]; item i runs on warp i (w_h > 1 implies n_items <= nw)
        const int i0 = s_wpre[ch], i1 = i0 + w_h - 1;
        const int wa = max(i0, cta_w0), wb = min(i1, cta_w0 + warps - 1);  // contributors inside this CTA
        bool carry = true;  // does this warp carry the head's state to the next level?
        if (wb > wa) {
            // level 1: several warps of this CTA share the head
            store_state(s_part + (size_t)warp * PART_FLOATS, M_, L_, A, lane);
            __syncwarp();
            int ticket = 0;
            if (lane == 0) ticket = atom_add_acq_rel_cta_shared(&s_cnt[wa - cta_w0], 1);
            ticket = __shfl_sync(0xffffffffu, ticket, 0);
            carry = (ticket == wb - wa);
            if (carry)
                merge_states<false>([&](int i) { return (const float *)(s_part + (size_t)(wa - cta_w0 + i) * PART_FLOATS); },
                                    wb - wa + 1, lane, M_, L_, A);
        }
        DBG_STAMP(9);  // level 1 done
        if (!carry) {
            DBG_FLUSH();
            continue;
        }
        const int cta_first = i0 / warps, cta_last = i1 / warps;
        if (cta_first == cta_last) {
            finalize_head(p, ch, M_, L_, A, lane);
            DBG_FLUSH();
            continue;
        }
        // level 2: several CTAs share the head.  A CTA holds at most one head that entered from the previous CTA
        // (slot 0) and one that continues into the next (slot 1).
        store_state(p.partials + ((size_t)blockIdx.x * 2 + ((i0 >= cta_w0) ? 1 : 0)) * PART_FLOATS, M_, L_, A, lane);
        __syncwarp();
        int ticket = 0;
        if (lane == 0) ticket = atom_add_acq_rel_gpu(p.counters + ch, 1);
        ticket = __shfl_sync(0xffffffffu, ticket, 0);
        DBG_STAMP(10);  // state published
        if (ticket == cta_last - cta_first) {  // last contributor: merge the CTA states
            merge_states<true>(
                [&](int i) {
                    const int c2 = cta_first + i;
                    return (const float *)(p.partials + ((size_t)c2 * 2 + ((i0 >= c2 * warps) ? 1 : 0)) * PART_FLOATS);
                },
                cta_last - cta_first + 1, lane, M_, L_, A);
            finalize_head(p, ch, M_, L_, A, lane);
            DBG_STAMP(11);  // head merged and written
            if (lane == 0) p.counters[ch] = 0;  // self-resetting for the next launch / graph replay
        }
        DBG_FLUSH();
    }
}

int launch_attend_mma(mpig_ctx *ctx, const AttendParams &p_in, cudaStream_t s, bool pdl) {
    AttendParams p = p_in;
    const int warps = ctx->attend.warps;
    MPIG_REQUIRE(warps >= 1 && warps <= 12, MPIG_EINVAL, "attend(mma): warps=%d outside [1,12]", warps);
    p.dbg = ctx->attend_debug ? ctx->dbg_buf : nullptr;
    p.skip = ctx->attend_skip;
    if (p.dbg) MPIG_CUDA(cudaMemsetAsync(p.dbg, 0, (size_t)ctx->max_partial_warps * 16 * sizeof(unsigned long long), s));
    const size_t smem = (size_t)warps * TILE * SLOT + (size_t)((warps + 1) & ~1) * 8 + (size_t)warps * 2 * PART_FLOATS * 4 + (size_t)warps * 4 +
                        (size_t)(p.H / p.Hq) * 4 + 2 * (size_t)(p.H + 1) * sizeof(int) + 16;
    MPIG_REQUIRE(smem <= 226 * 1024, MPIG_EINVAL, "attend(mma): warps=%d H=%d needs %zu B shared memory (> 227 KB)", warps, p.H, smem);
    MPIG_FUNC_ATTR((attend_mma_kernel<true, false>), cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    MPIG_FUNC_ATTR((attend_mma_kernel<false, false>), cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    MPIG_FUNC_ATTR((attend_mma_kernel<true, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    MPIG_FUNC_ATTR((attend_mma_kernel<false, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    int ctas = ctx->attend.ctas;
    if (ctas <= 0) {
        const int occ = (int)std::max<size_t>(1, std::min<size_t>((227 * 1024) / (smem + 1024), 2048 / (warps * 32)));
        ctas = ctx->num_sms * occ;
    }
    MPIG_REQUIRE(ctas * 2 <= ctx->max_partial_warps * 2, MPIG_EINVAL, "attend(mma): %d CTAs exceed partial scratch", ctas);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(ctas);
    cfg.blockDim = dim3(warps * 32);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    if (p.dbg) {
        if (ctx->attend.tma) MPIG_CUDA(cudaLaunchKernelEx(&cfg, attend_mma_kernel<true, true>, p));
        else MPIG_CUDA(cudaLaunchKernelEx(&cfg, attend_mma_kernel<false, true>, p));
    } else if (ctx->attend.tma) MPIG_CUDA(cudaLaunchKernelEx(&cfg, attend_mma_kernel<true, false>, p));
    else MPIG_CUDA(cudaLaunchKernelEx(&cfg, attend_mma_kernel<false, false>, p));
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

}  // namespace mpig
