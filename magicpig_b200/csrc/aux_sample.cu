// aux_sample.cu -- temperature / top-p sampling of a batch's fp32 logits on the device (see include/magicpig_b200_aux.h).
//
// Stands in for the reference caller's topp_temperature_decode (models/utils.py:57-100) and its argmax for temperature < 0.1
// (models/llama.py:340-343).  One launch samples one token for each of B rows.  Contract for row b, logits l_i (i < V),
// T = temperature[b], p = top_p[b]:
//   * invalid row: any l_i NaN or +inf, or no finite l_i  ->  token 0 and bit (b % 32) of status[b / 32] is set.
//   * greedy, T <= 0 (or NaN): the smallest i with l_i == max l (torch.argmax's first occurrence).
//   * weights, T > 0: w_i = exp2f((l_i - m) * k) in fp32 with m = max l and k = 1.44269504f / T (fp32 division), both
//     products rounded to nearest; -inf logits get w_i = 0.  w_i <= 1 and w_i == 1 at the max.  Fixed point:
//     W_i = floor(w_i * 2^40) (exact: a power-of-two scale, then truncation), S = sum W_i < V * 2^41.  From here on integer.
//   * nucleus: order the tokens by W descending, ties by lower index first; token i is kept iff the sum of the W of the tokens
//     ordered before it is <= floor(p * S), computed exactly from p's 24-bit significand times S in 128 bits.  p >= 1 keeps
//     every token, p <= 0 (or NaN) only the first in that order.  This is the reference's `cumsum > top_p` shifted by one, with
//     the order of tied probabilities made definite.
//   * draw: r = x | y << 32 of curand_Philox4x32_10(counter (offset lo, offset hi, b, 0), key (seed lo, seed hi)) = (x, y, ..),
//     target = umulhi64(r, S_keep) with S_keep the kept mass; the token is the kept index, in INDEX order, at which the running
//     kept sum first exceeds target.  The kernel reads *offset and never writes it.
// Every stage after the fp32 weights is integer arithmetic, so the result is bitwise deterministic and independent of how the
// row is split across CTAs.
//
// Layout: one cluster of C <= 8 CTAs per row; CTA `rank` stages the contiguous slice [rank * slice, +slice) of the row in shared
// memory (fp32 logits, then in place the 32-bit keys below), so HBM is read once and every later pass runs from SMEM.  Cluster
// reductions go through distributed shared memory: each CTA publishes its partial in its own SMEM, cluster.sync(), and every CTA
// combines the C partials in rank order, so all CTAs hold the same integers.  Exchange slots alternate between two buffers, so one
// cluster barrier per exchange suffices.
//   A  max with its first index, and the invalid flag
//   B  S
//   R  up to 4 radix passes of 256-bin (count, u64 mass) histograms that select the nucleus threshold value W*
//   E  per CTA: mass and count above W*, and ties at W* -> tie ranks in CTA order (= index order) and the kept mass per CTA
// The CTA holding target then scans its slice in index order (one warp per contiguous segment).
//
// Radix key: key(W) = bits of (float)W.  (float)W is exact (W < 2^24, or W = w * 2^40 with w's 24-bit significand), and positive
// floats order like their bits, so the 32-bit key orders the W and determines W; 4 passes of 8 bits decide it.
//
// Speculative sampling (mpig_aux_verify_sample) runs the same kernel as sample_kernel<true> over the B*T rows of a verification
// step, row (b, t) checking the draft d = ids[b, t + 1] (t <= T - 2):
//   * greedy: accept iff d is the first argmax; sampled: accept iff d is kept and umulhi64(r_acc, S_keep) < W_d, r_acc from
//     Philox counter (offset lo, offset hi, b, t + 1) -- probability p(d);
//   * the row's final token if acceptance ends here: the argmax (greedy), or the draw above with word (.., b, 0) over the kept set
//     without d (mass S_keep - W_d if d is kept), scanned in index order with d's weight 0; with no draft it is the plain draw.
// verify_resolve_kernel then takes k = the first rejected row (T - 1 if none): the request emits d_1 .. d_k and row k's final
// token.  For a one-hot draft every emitted token follows the row's nucleus distribution; T = 1 is mpig_aux_sample bit for bit.
#include <cooperative_groups.h>
#include <curand_philox4x32_x.h>

#include "../../include/magicpig_b200_aux.h"
#include "common.cuh"

namespace cg = cooperative_groups;

namespace mpig {

constexpr int SMP_THREADS = 512;
constexpr int SMP_WARPS = SMP_THREADS / 32;
constexpr int SMP_MAX_C = 8;                     // portable cluster size
constexpr int SMP_SLICE_ALIGN = 256;             // slice length granule (elements)
constexpr int SMP_ROWS_PER_CTA_HINT = 4096;      // C = ceil(V / this), at most SMP_MAX_C
constexpr int SMP_SMEM_CAP = 200 * 1024;         // dynamic shared memory of one slice (bytes)
constexpr int SMP_MAX_EOS = 8;
constexpr int SMP_MAX_VERIFY_T = 8;               // rows per request of mpig_aux_verify_sample

struct SampleParams {
    const float *logits;
    long long ld;
    int V, C, slice;
    const float *temperature, *top_p;
    unsigned long long seed;
    const unsigned long long *offset;
    long long *ids_out;
    long long ids_stride;
    int *tokens_out, *count, *done;
    int max_new, n_eos;
    int eos[SMP_MAX_EOS];
    int *status;
    long long *dbg;   // (B, 5): S, floor(p S), S_keep, kept count, target; verification: (B, T, 9), see mpig_aux_verify_sample
    float *dbg_w;     // (B, V): w_i; verification: (B, T, V)
    // verification (sample_kernel<true> and verify_resolve_kernel): row (b, t) at logits + b * ld + t * ld_t, its draft at
    // ids_out[b * ids_stride + t + 1]; rows (B, T, 2) receives each row's final token and flags
    int T;
    long long ld_t;
    int *rows;
    int *drop, *limit, *steps, *accepted;
    long long hist_ld;
    // filters (sample_kernel<.., true>, verify_resolve_kernel<true>): per-request (B,) arrays and the penalty table (B, tab_ld)
    const int *top_k;
    const float *min_p, *rep, *pres, *freq;
    unsigned *tab;
    long long tab_ld;
};

constexpr int ROW_ACCEPT = 1, ROW_INVALID = 2;   // flags of a verification row

__device__ __forceinline__ unsigned long long key_weight(unsigned key) { return __float2ull_rz(__uint_as_float(key)); }
__device__ __forceinline__ float row_weight(float l, float mx, float k) { return exp2f((l - mx) * k); }
__device__ __forceinline__ unsigned long long fixed_weight(float w) { return __float2ull_rz(w * 0x1p40f); }
__device__ __forceinline__ unsigned long long philox_word(unsigned long long off, int b, unsigned word, unsigned long long seed) {
    const uint4 rnd = curand_Philox4x32_10(make_uint4((unsigned)off, (unsigned)(off >> 32), (unsigned)b, word),
                                           make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
    return (unsigned long long)rnd.x | ((unsigned long long)rnd.y << 32);
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ unsigned long long warp_incl_scan_u64(unsigned long long v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// sum over the CTA, returned to every thread (two barriers; scratch has SMP_WARPS entries)
__device__ __forceinline__ unsigned long long block_sum_u64(unsigned long long v, unsigned long long *scratch) {
    v = warp_sum_u64(v);
    __syncthreads();   // scratch may still be read by a previous call
    if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
    __syncthreads();
    unsigned long long t = 0;
#pragma unroll
    for (int w = 0; w < SMP_WARPS; ++w) t += scratch[w];
    return t;
}

// exact floor(p * S) for 0 < p < 1: p = m24 * 2^(e - 24) with m24 its 24-bit significand
__device__ __forceinline__ unsigned long long nucleus_threshold(float p, unsigned long long S) {
    if (p >= 1.f) return S;
    if (!(p > 0.f)) return 0;
    int e = 0;
    const float mant = frexpf(p, &e);   // p = mant * 2^e, mant in [0.5, 1), e <= 0
    const unsigned long long m24 = (unsigned long long)(mant * 16777216.f);
    const unsigned long long lo = m24 * S, hi = __umul64hi(m24, S);
    const int sh = 24 - e;   // >= 24
    if (sh >= 128) return 0;
    if (sh >= 64) return hi >> (sh - 64);
    return (lo >> sh) | (hi << (64 - sh));
}

// ---- filters (FILT): the per-row values as the device reads them, the penalties, and the selects behind top-k and top-p ----
struct RowFilters {
    int top_k;
    float min_p, r, f, pr;
    bool pen;   // some penalty is not neutral: the row reads its table slice
};

__device__ __forceinline__ RowFilters row_filters(const SampleParams &p, int b) {
    RowFilters q;
    q.top_k = p.top_k[b];
    q.min_p = p.min_p[b];   // nucleus_threshold(min_p, 2^40): NaN or <= 0 -> 0 (off), >= 1 -> 2^40
    const float r = p.rep[b], f = p.freq[b], pr = p.pres[b];
    q.r = isfinite(r) && r > 0.f ? r : 1.f;
    q.f = isfinite(f) ? f : 0.f;
    q.pr = isfinite(pr) ? pr : 0.f;
    q.pen = !(q.r == 1.f && q.f == 0.f && q.pr == 0.f);
    return q;
}

// The drafts d_1 .. d_t that a verification row's prefix emits (ids[b, 1 .. t]; an id outside [0, V) is no token), -1 beyond t.
__device__ const int *row_drafts(const SampleParams &p, int b, int t) {
    __shared__ int drafts[SMP_MAX_VERIFY_T];
    if (threadIdx.x < SMP_MAX_VERIFY_T) {
        int d = -1;
        if ((int)threadIdx.x < t) {
            const long long id = p.ids_out[(size_t)b * p.ids_stride + 1 + threadIdx.x];
            d = id >= 0 && id < p.V ? (int)id : -1;
        }
        drafts[threadIdx.x] = d;
    }
    __syncthreads();
    return drafts;
}

// The penalised logit l3 of token i: e = its table entry, extra = the drafts before the row that equal i.  fp32, every operation
// rounded to nearest with no contraction, so numpy float32 restates it bit for bit.
__device__ __forceinline__ float penalise(float l, unsigned e, unsigned extra, const RowFilters &q) {
    const unsigned c = (e & 0x7FFFFFFFu) + extra;
    const bool seen = (e >> 31) || c > 0;
    const float l1 = seen ? (l > 0.f ? __fdiv_rn(l, q.r) : __fmul_rn(l, q.r)) : l;
    const float l2 = __fsub_rn(l1, __fmul_rn(q.f, __uint2float_rn(c)));
    return c > 0 ? __fsub_rn(l2, q.pr) : l2;
}

__device__ __forceinline__ unsigned draft_count(const int *drafts, int t, int i) {
    unsigned c = 0;
    for (int j = 0; j < t; ++j) c += drafts[j] == i;
    return c;
}

// the penalised logit of the draft d a verification row checks, recomputed bitwise as stage A staged it
__device__ __forceinline__ float draft_logit(const float *row, int d, const unsigned *tab, const int *drafts, int t,
                                             const RowFilters &q) {
    const float l = __ldg(row + d);
    return q.pen ? penalise(l, tab[d], draft_count(drafts, t, d), q) : l;
}

// min over the CTA, returned to every thread (two barriers; scratch has SMP_WARPS entries)
__device__ __forceinline__ unsigned block_min_u32(unsigned v, unsigned long long *scratch) {
    v = __reduce_min_sync(0xffffffffu, v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
    __syncthreads();
    unsigned m = UINT_MAX;
#pragma unroll
    for (int w = 0; w < SMP_WARPS; ++w) m = min(m, (unsigned)scratch[w]);
    return m;
}

// Stage B of a filtered row: the weights and keys in place of the penalised logits, S, and for min-p the count n_m of tokens with
// W >= Wm and the smallest key v_m among them, all cluster-wide.
struct Weighed {
    unsigned long long S, n_m;
    unsigned v_m;
};

__device__ Weighed filtered_weights(const cg::cluster_group &cl, unsigned *sbuf, int n, int C, float mx, float k,
                                    unsigned long long Wm, float *dbg_w, unsigned long long *scratch) {
    __shared__ unsigned long long x_s, x_n;
    __shared__ unsigned x_v;
    const int tid = threadIdx.x, lane = tid & 31;
    const float *slf = reinterpret_cast<const float *>(sbuf);
    unsigned long long s = 0, cnt = 0;
    unsigned vm = UINT_MAX;
    for (int i = tid; i < n; i += SMP_THREADS) {
        const float w = row_weight(slf[i], mx, k);
        const unsigned long long W = fixed_weight(w);
        const unsigned key = __float_as_uint(__ull2float_rn(W));
        sbuf[i] = key;
        s += W;
        if (W >= Wm) { ++cnt; vm = min(vm, key); }
        if (dbg_w) dbg_w[i] = w;
    }
    s = block_sum_u64(s, scratch);
    cnt = block_sum_u64(cnt, scratch);
    vm = block_min_u32(vm, scratch);
    if (tid == 0) { x_s = s; x_n = cnt; x_v = vm; }
    cl.sync();
    Weighed o;
    unsigned long long rs = 0, rn = 0;
    unsigned rv = UINT_MAX;
    if (lane < C) {
        rs = *cl.map_shared_rank(&x_s, lane);
        rn = *cl.map_shared_rank(&x_n, lane);
        rv = *cl.map_shared_rank(&x_v, lane);
    }
    o.S = warp_sum_u64(rs);
    o.n_m = warp_sum_u64(rn);
    o.v_m = __reduce_min_sync(0xffffffffu, rv);
    return o;
}

// One radix select over the cluster's keys: 4 passes of 8 bits with the (count, mass) histograms of the top-p select, exchanged
// through the same alternating buffers (a select has an even number of passes, so consecutive selects keep alternating).
// BY_COUNT: the key of the goal-th token of the order (1 <= goal <= V); otherwise the smallest present key whose strictly greater
// mass is <= goal.  Returns the key; above_m / above_c: the mass and count of the keys above it; at: the tokens holding it.
template <bool BY_COUNT>
__device__ unsigned radix_select(const cg::cluster_group &cl, const unsigned *keys, int n, int C, unsigned long long goal,
                                 unsigned (*hmass)[3][256], unsigned (*hcount)[256], unsigned long long *mmass, unsigned *mcount,
                                 unsigned long long &above_m, unsigned long long &above_c, unsigned long long &at) {
    __shared__ unsigned long long scan_m[SMP_WARPS], scan_c[SMP_WARPS], sel_m, sel_c, sel_n;
    __shared__ int sel;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned v = 0;
    above_m = above_c = at = 0;
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        unsigned (*hm)[256] = hmass[pass & 1];
        unsigned *hc = hcount[pass & 1];
        if (tid < 256) { hm[0][tid] = 0; hm[1][tid] = 0; hm[2][tid] = 0; hc[tid] = 0; }
        __syncthreads();
        for (int i0 = 0; i0 < n; i0 += SMP_THREADS) {
            const int i = i0 + tid;
            const unsigned key = i < n ? keys[i] : 0u;
            const bool ok = i < n && (pass == 0 || (key >> (shift + 8)) == (v >> (shift + 8)));
            const unsigned bin = ok ? (key >> shift) & 255u : 256u;
            const unsigned long long W = ok ? key_weight(key) : 0ull;
            const unsigned grp = __match_any_sync(0xffffffffu, bin);
            if (grp == 0xffffffffu) {
                const unsigned long long m = warp_sum_u64(W);
                if (lane == 0 && ok) {
                    atomicAdd(&hc[bin], 32u);
                    atomicAdd(&hm[0][bin], (unsigned)(m & 0xFFFFu));
                    atomicAdd(&hm[1][bin], (unsigned)((m >> 16) & 0xFFFFu));
                    atomicAdd(&hm[2][bin], (unsigned)(m >> 32));
                }
            } else if (ok) {
                atomicAdd(&hc[bin], 1u);
                atomicAdd(&hm[0][bin], (unsigned)(W & 0xFFFFu));
                atomicAdd(&hm[1][bin], (unsigned)((W >> 16) & 0xFFFFu));
                atomicAdd(&hm[2][bin], (unsigned)(W >> 32));
            }
        }
        cl.sync();
        if (tid < 256) {
            unsigned long long mass = 0;
            unsigned cnt = 0;
            for (int r = 0; r < C; ++r) {
                const unsigned(*pm)[256] = cl.map_shared_rank(hm, r);
                mass += (unsigned long long)pm[0][tid] + ((unsigned long long)pm[1][tid] << 16) + ((unsigned long long)pm[2][tid] << 32);
                cnt += cl.map_shared_rank(hc, r)[tid];
            }
            mmass[tid] = mass;
            mcount[tid] = cnt;
        }
        if (tid == 0) sel = BY_COUNT ? -1 : 256;
        __syncthreads();
        // suffix sums over the bins in descending order: thread t < 256 takes bin 255 - t
        if (tid < 256) {
            const int bin = 255 - tid;
            const unsigned long long m = mmass[bin], c = mcount[bin];
            const unsigned long long im = warp_incl_scan_u64(m, lane), ic = warp_incl_scan_u64(c, lane);
            if (lane == 31) { scan_m[warp] = im; scan_c[warp] = ic; }
            __syncwarp();
            asm volatile("bar.sync 1, 256;" ::: "memory");
            unsigned long long bm = 0, bc = 0;
            for (int w = 0; w < warp; ++w) { bm += scan_m[w]; bc += scan_c[w]; }
            const unsigned long long em = bm + im - m, ec = bc + ic - c;   // mass / count of the bins above `bin`
            if (c > 0) {
                if (BY_COUNT) {
                    if (above_c + ec + c >= goal) atomicMax(&sel, bin);
                } else if (above_m + em <= goal) {
                    atomicMin(&sel, bin);
                }
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            if (bin == sel) { sel_m = em; sel_c = ec; sel_n = c; }
        }
        __syncthreads();
        above_m += sel_m;
        above_c += sel_c;
        at = sel_n;
        v |= (unsigned)sel << shift;
    }
    return v;
}

template <bool FILT>
__device__ void sample_commit(const SampleParams &p, int b, int token) {
    if (p.ids_out) p.ids_out[(size_t)b * p.ids_stride] = token;
    if (p.tokens_out && !p.done[b]) {
        int c = p.count[b];
        if (c < p.max_new) {
            p.tokens_out[(size_t)b * p.max_new + c] = token;
            p.count[b] = ++c;
            if constexpr (FILT) p.tab[(size_t)b * p.tab_ld + token] += 1u;
        }
        bool eos = false;
        for (int k = 0; k < p.n_eos; ++k) eos |= token == p.eos[k];
        if (eos || c >= p.max_new) p.done[b] = 1;
    }
}

// VERIFY = false: mpig_aux_sample, one row per request.  VERIFY = true: the rows of mpig_aux_verify_sample, row (b, t) with draft
// d = ids[b, t + 1] (t < T - 1; none on the last row, and an id outside [0, V) is no token): the same stages decide whether d is
// accepted and draw the row's final token from the kept set without d (the residual), scanning in index order with d's weight
// taken as 0.  The row's accept bit and final token go to p.rows; verify_resolve_kernel does the bookkeeping.
//
// FILT = true: the filtered rule of mpig_aux_sample_filtered / mpig_aux_verify_sample_filtered (include/magicpig_b200_aux.h).  Stage
// A stages the penalised logits (a verification row counts its drafts d_1 .. d_t too), stage B also counts min-p's tokens, top-k is
// a count select and top-p a mass select with thr = floor(p S_k) over the same histograms, and the kept set is the first
// K = max(1, min(n_k, n_p, n_m)) tokens of the order: v* is the key of the K-th token and K - (tokens above v*) ties at v* are kept.
// Everything after v* is the unfiltered code.  FILT = false compiles to the kernel of the unfiltered calls unchanged.
template <bool VERIFY, bool FILT>
__global__ void __launch_bounds__(SMP_THREADS) sample_kernel(const __grid_constant__ SampleParams p) {
    extern __shared__ __align__(16) unsigned sbuf[];   // the slice: fp32 logits, then their keys
    // radix histograms (exchanged), alternating buffers.  The mass of a bin is kept as three u32 parts (bits 0-15, 16-31, 32-):
    // a 64-bit shared atomic add is a compare-and-swap loop on sm_90, the 32-bit one a native atomic.  A part gains < 2^16 per
    // add and a slice holds < 2^16 elements, so no part overflows.
    __shared__ unsigned hmass[2][3][256];
    __shared__ unsigned hcount[2][256];
    __shared__ unsigned long long mmass[256];          // merged histogram of the current pass (local)
    __shared__ unsigned mcount[256];
    __shared__ unsigned long long scratch[SMP_WARPS], wscan[SMP_WARPS];
    __shared__ unsigned long long xb_s, xe_mass;       // exchanges B, E
    __shared__ unsigned xe_count, xe_ties, xe_ties_d;
    __shared__ float xa_max, red_max[SMP_WARPS];       // exchange A
    __shared__ int xa_idx, xa_bad, red_idx[SMP_WARPS];
    __shared__ int sel_bin, sel_warp;
    __shared__ unsigned long long sel_excl, sel_prefix, sel_tie_base;

    cg::cluster_group cl = cg::this_cluster();
    const int C = p.C, rank = (int)cl.block_rank(), rw = blockIdx.x / C;
    const int b = VERIFY ? rw / p.T : rw, t = VERIFY ? rw % p.T : 0;
    const int lo = rank * p.slice, n = max(0, min(p.slice, p.V - lo));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float *slf = reinterpret_cast<float *>(sbuf);
    const float *row = p.logits + (size_t)b * p.ld + (VERIFY ? (size_t)t * p.ld_t : 0);
    const float *src = row + lo;
    int d = -1;   // the draft this row checks
    if (VERIFY && t < p.T - 1) {
        const long long id = p.ids_out[(size_t)b * p.ids_stride + t + 1];
        d = id >= 0 && id < p.V ? (int)id : -1;
    }
    constexpr int DBG_N = VERIFY ? (FILT ? 12 : 9) : (FILT ? 8 : 5);   // debug integers per row
    RowFilters fr{};
    const int *drafts = nullptr;
    const unsigned *tab = nullptr;
    if constexpr (FILT) {
        fr = row_filters(p, b);
        drafts = row_drafts(p, b, t);
        tab = p.tab + (size_t)b * p.tab_ld;
    }

    // ---- A: stage the slice; max with its first index; invalid flag ----
    float mx = -INFINITY;
    int mi = INT_MAX, bad = 0;
    if constexpr (FILT) {   // the penalised logits; a NaN or +inf raw or penalised logit makes the row invalid
        for (int i = tid; i < n; i += SMP_THREADS) {
            float v = __ldg(src + i);
            if (!(v < INFINITY)) bad = 1;
            if (fr.pen) v = penalise(v, tab[lo + i], draft_count(drafts, t, lo + i), fr);
            slf[i] = v;
            if (!(v < INFINITY)) bad = 1;
            else if (v > mx || mi == INT_MAX) { mx = v; mi = lo + i; }
        }
    } else {
        for (int i = tid; i < n; i += SMP_THREADS) {
            const float v = __ldg(src + i);
            slf[i] = v;
            if (!(v < INFINITY)) bad = 1;   // NaN or +inf
            else if (v > mx || mi == INT_MAX) { mx = v; mi = lo + i; }   // indices rise within a thread: first occurrence
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, mx, o);
        const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
        if (om > mx || (om == mx && oi < mi)) { mx = om; mi = oi; }
    }
    if (lane == 0) { red_max[warp] = mx; red_idx[warp] = mi; }
    bad = __syncthreads_or(bad);
    if (tid == 0) {
        for (int w = 1; w < SMP_WARPS; ++w)
            if (red_max[w] > mx || (red_max[w] == mx && red_idx[w] < mi)) { mx = red_max[w]; mi = red_idx[w]; }
        xa_max = mx; xa_idx = mi; xa_bad = bad;
    }
    cl.sync();
    {   // every warp combines the C partials (lane r reads rank r); rank order, same rule -> the same result everywhere
        float om = -INFINITY;
        int oi = INT_MAX, ob = 0;
        if (lane < C) {
            om = *cl.map_shared_rank(&xa_max, lane);
            oi = *cl.map_shared_rank(&xa_idx, lane);
            ob = *cl.map_shared_rank(&xa_bad, lane);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const float tm = __shfl_xor_sync(0xffffffffu, om, o);
            const int ti = __shfl_xor_sync(0xffffffffu, oi, o);
            if (tm > om || (tm == om && ti < oi)) { om = tm; oi = ti; }
        }
        mx = om; mi = oi;
        bad = __any_sync(0xffffffffu, ob) || !(mx > -INFINITY);
    }
    const float T = p.temperature[b], top_p = p.top_p[b];
    if (bad || !(T > 0.f)) {
        if (rank == 0 && tid == 0) {
            const int token = bad ? 0 : mi;
            if constexpr (VERIFY) {
                const bool acc = !bad && d == mi;
                p.rows[2 * rw] = token;
                p.rows[2 * rw + 1] = (bad ? ROW_INVALID : 0) | (acc ? ROW_ACCEPT : 0);
                if (p.dbg) {
                    long long *dd = p.dbg + (size_t)rw * DBG_N;
                    for (int j = 0; j < DBG_N; ++j) dd[j] = 0;
                    dd[3] = bad ? 0 : 1;
                    dd[6] = acc;
                }
            } else {
                if (bad && p.status) atomicOr(p.status + (b >> 5), 1 << (b & 31));
                sample_commit<FILT>(p, b, token);
                if (p.dbg) {
                    long long *d = p.dbg + (size_t)b * DBG_N;
                    d[0] = d[1] = d[2] = d[4] = 0;
                    d[3] = bad ? 0 : 1;
                    if constexpr (FILT) d[5] = d[6] = d[7] = 0;
                }
            }
        }
        cl.sync();   // no CTA leaves while a peer may still read its exchange slot
        return;
    }

    // ---- B: weights, their keys in place of the logits, S ----
    const float k = 1.44269504f / T;
    unsigned long long S, thr;
    unsigned vstar = 0;              // p >= 1: every token is kept (W* = 0: every zero-weight tie kept too)
    unsigned long long above = 0;    // mass of the keys above the decided prefix
    unsigned long long kept_n = 0, n_k = 0, S_k = 0, n_m = 0;   // FILT: K, top-k's count and mass, min-p's count
    if constexpr (FILT) {
        const Weighed wb = filtered_weights(cl, sbuf, n, C, mx, k, nucleus_threshold(fr.min_p, 1ull << 40),
                                            p.dbg_w ? p.dbg_w + (size_t)rw * p.V + lo : nullptr, scratch);
        S = wb.S;
        n_m = wb.n_m;
        // top-k: the key of the n_k-th token by a count select; S_k the mass of the first n_k tokens (v = 0 stands for all V)
        unsigned v_k = 0, v_p = 0;
        n_k = p.V;
        S_k = S;
        if (fr.top_k > 0 && fr.top_k < p.V) {
            unsigned long long am, ac, at;
            n_k = (unsigned long long)fr.top_k;
            v_k = radix_select<true>(cl, sbuf, n, C, n_k, hmass, hcount, mmass, mcount, am, ac, at);
            S_k = am + (n_k - ac) * key_weight(v_k);
        }
        // top-p over the top-k set: positions j < n_k whose mass before is <= floor(p S_k), a prefix of n_p tokens
        thr = nucleus_threshold(top_p, S_k);
        unsigned long long n_p = p.V;
        if (top_p < 1.f) {
            unsigned long long am, ac, at;
            v_p = radix_select<false>(cl, sbuf, n, C, thr, hmass, hcount, mmass, mcount, am, ac, at);
            const unsigned long long Wp = key_weight(v_p);
            n_p = ac + (Wp > 0 ? min(at, (thr - am) / Wp + 1) : at);
        }
        kept_n = max(1ull, min(min(n_k, n_p), n_m));
        vstar = kept_n == n_p ? v_p : kept_n == n_k ? v_k : wb.v_m;
    } else {
    unsigned long long s_loc = 0;
    for (int i = tid; i < n; i += SMP_THREADS) {
        const float w = row_weight(slf[i], mx, k);
        const unsigned long long W = fixed_weight(w);
        sbuf[i] = __float_as_uint(__ull2float_rn(W));
        s_loc += W;
        if (p.dbg_w) p.dbg_w[(size_t)rw * p.V + lo + i] = w;
    }
    s_loc = block_sum_u64(s_loc, scratch);
    if (tid == 0) xb_s = s_loc;
    cl.sync();
    S = lane < C ? *cl.map_shared_rank(&xb_s, lane) : 0ull;
    S = warp_sum_u64(S);
    thr = nucleus_threshold(top_p, S);

    // ---- R: the threshold key v* = the smallest present key whose strictly-greater mass is <= thr ----
    if (top_p < 1.f) {
        for (int pass = 0; pass < 4; ++pass) {
            const int shift = 24 - 8 * pass;
            unsigned (*hm)[256] = hmass[pass & 1];
            unsigned *hc = hcount[pass & 1];
            if (tid < 256) { hm[0][tid] = 0; hm[1][tid] = 0; hm[2][tid] = 0; hc[tid] = 0; }
            __syncthreads();
            for (int i0 = 0; i0 < n; i0 += SMP_THREADS) {
                const int i = i0 + tid;
                const unsigned key = i < n ? sbuf[i] : 0u;
                const bool ok = i < n && (pass == 0 || (key >> (shift + 8)) == (vstar >> (shift + 8)));
                const unsigned bin = ok ? (key >> shift) & 255u : 256u;
                const unsigned long long W = ok ? key_weight(key) : 0ull;
                const unsigned grp = __match_any_sync(0xffffffffu, bin);
                if (grp == 0xffffffffu) {   // the whole warp in one bin (flat or tied rows): one atomic pair
                    const unsigned long long m = warp_sum_u64(W);
                    if (lane == 0 && ok) {   // m < 2^46: its parts are < 2^16, < 2^16 and < 2^14
                        atomicAdd(&hc[bin], 32u);
                        atomicAdd(&hm[0][bin], (unsigned)(m & 0xFFFFu));
                        atomicAdd(&hm[1][bin], (unsigned)((m >> 16) & 0xFFFFu));
                        atomicAdd(&hm[2][bin], (unsigned)(m >> 32));
                    }
                } else if (ok) {
                    atomicAdd(&hc[bin], 1u);
                    atomicAdd(&hm[0][bin], (unsigned)(W & 0xFFFFu));
                    atomicAdd(&hm[1][bin], (unsigned)((W >> 16) & 0xFFFFu));
                    atomicAdd(&hm[2][bin], (unsigned)(W >> 32));
                }
            }
            cl.sync();
            unsigned long long mass = 0;
            unsigned cnt = 0;
            if (tid < 256) {
                for (int r = 0; r < C; ++r) {
                    const unsigned(*pm)[256] = cl.map_shared_rank(hm, r);
                    mass += (unsigned long long)pm[0][tid] + ((unsigned long long)pm[1][tid] << 16) + ((unsigned long long)pm[2][tid] << 32);
                    cnt += cl.map_shared_rank(hc, r)[tid];
                }
                mmass[tid] = mass;
                mcount[tid] = cnt;
            }
            if (tid == 0) sel_bin = 256;
            __syncthreads();
            // suffix sums over the bins in descending order: thread t < 256 takes bin 255 - t
            if (tid < 256) {
                const int bin = 255 - tid;
                const unsigned long long m = mmass[bin];
                const unsigned long long incl = warp_incl_scan_u64(m, lane);
                if (lane == 31) wscan[warp] = incl;
                __syncwarp();
                asm volatile("bar.sync 1, 256;" ::: "memory");
                unsigned long long base = 0;
                for (int w = 0; w < warp; ++w) base += wscan[w];
                const unsigned long long excl = base + incl - m;   // mass of the bins above `bin`
                if (mcount[bin] > 0 && above + excl <= thr) atomicMin(&sel_bin, bin);
                asm volatile("bar.sync 1, 256;" ::: "memory");
                if (bin == sel_bin) sel_excl = excl;
            }
            __syncthreads();
            above += sel_excl;
            vstar |= (unsigned)sel_bin << shift;
        }
    }
    }
    const unsigned long long Wstar = key_weight(vstar);

    // ---- E: per CTA mass / count above v* and ties at v*; kept mass per CTA; target ----
    unsigned long long gmass = 0;
    unsigned gcount = 0, ties = 0, ties_d = 0;
    for (int i = tid; i < n; i += SMP_THREADS) {
        const unsigned key = sbuf[i];
        if (key > vstar) { gmass += key_weight(key); ++gcount; }
        else if (key == vstar) {
            ++ties;
            if (VERIFY && lo + i < d) ++ties_d;   // ties ranked before the draft
        }
    }
    gmass = block_sum_u64(gmass, scratch);
    gcount = (unsigned)block_sum_u64(gcount, scratch);
    ties = (unsigned)block_sum_u64(ties, scratch);
    if (VERIFY) ties_d = (unsigned)block_sum_u64(ties_d, scratch);
    if (tid == 0) {
        xe_mass = gmass; xe_count = gcount; xe_ties = ties;
        if (VERIFY) xe_ties_d = ties_d;
    }
    cl.sync();
    // lane r < C: rank r's numbers (every warp computes the same)
    unsigned long long r_mass = 0;
    unsigned r_count = 0, r_ties = 0, r_ties_d = 0;
    if (lane < C) {
        r_mass = *cl.map_shared_rank(&xe_mass, lane);
        r_count = *cl.map_shared_rank(&xe_count, lane);
        r_ties = *cl.map_shared_rank(&xe_ties, lane);
        if (VERIFY) r_ties_d = *cl.map_shared_rank(&xe_ties_d, lane);
    }
    const unsigned long long ties_total = warp_sum_u64(r_ties);
    const unsigned long long ties_before = warp_incl_scan_u64(r_ties, lane) - r_ties;
    const unsigned long long keep_ties = FILT ? kept_n - warp_sum_u64(r_count)
                                              : (Wstar > 0 ? min(ties_total, (thr - above) / Wstar + 1) : ties_total);
    const unsigned long long r_keep_ties = keep_ties > ties_before ? min(keep_ties - ties_before, (unsigned long long)r_ties) : 0ull;
    const unsigned long long r_kept = r_mass + r_keep_ties * Wstar;
    const unsigned long long S_keep = warp_sum_u64(r_kept);
    const unsigned long long kept_count = warp_sum_u64(r_count + r_keep_ties);
    // the draft's weight (recomputed from its logit by every thread, bitwise as staged) and keep bit; the residual mass per rank
    unsigned long long W_d = 0;
    bool kept_d = false;
    if (VERIFY && d >= 0) {
        W_d = fixed_weight(row_weight(FILT ? draft_logit(row, d, tab, drafts, t, fr) : __ldg(row + d), mx, k));
        const unsigned key_d = __float_as_uint(__ull2float_rn(W_d));
        kept_d = key_d > vstar || (key_d == vstar && warp_sum_u64(r_ties_d) < keep_ties);
    }
    const unsigned long long r_res = VERIFY && kept_d && lane == d / p.slice ? r_kept - W_d : r_kept;
    const unsigned long long S_res = VERIFY && kept_d ? S_keep - W_d : S_keep;
    const unsigned long long r_prefix = warp_incl_scan_u64(r_res, lane) - r_res;
    const unsigned long long off = *p.offset;
    const unsigned long long r64 = philox_word(off, b, 0u, p.seed);
    const unsigned long long target = __umul64hi(r64, S_res);
    const unsigned holder = __ballot_sync(0xffffffffu, lane < C && r_prefix <= target && target < r_prefix + r_res);
    const int sel_rank = __ffs(holder) - 1;
    if constexpr (VERIFY) {
        if (rank == 0 && tid == 0) {
            const unsigned long long acc_target = d >= 0 ? __umul64hi(philox_word(off, b, (unsigned)t + 1u, p.seed), S_keep) : 0ull;
            const bool acc = kept_d && acc_target < W_d;
            p.rows[2 * rw + 1] = acc ? ROW_ACCEPT : 0;
            if (!holder) p.rows[2 * rw] = mi;   // S_res = 0: d holds all the kept mass and is accepted for sure
            if (p.dbg) {
                long long *dd = p.dbg + (size_t)rw * DBG_N;
                dd[0] = (long long)S; dd[1] = (long long)thr; dd[2] = (long long)S_keep; dd[3] = (long long)kept_count;
                dd[4] = (long long)__umul64hi(r64, S_keep);
                dd[5] = (long long)W_d; dd[6] = kept_d; dd[7] = (long long)acc_target; dd[8] = (long long)S_res;
                if constexpr (FILT) { dd[9] = (long long)n_k; dd[10] = (long long)S_k; dd[11] = (long long)n_m; }
            }
        }
    } else if (rank == 0 && tid == 0 && p.dbg) {
        long long *d = p.dbg + (size_t)b * DBG_N;
        d[0] = (long long)S; d[1] = (long long)thr; d[2] = (long long)S_keep; d[3] = (long long)kept_count; d[4] = (long long)target;
        if constexpr (FILT) { d[5] = (long long)n_k; d[6] = (long long)S_k; d[7] = (long long)n_m; }
    }

    if (rank == sel_rank) {
        const unsigned long long my_keep_ties = __shfl_sync(0xffffffffu, r_keep_ties, sel_rank);
        const unsigned long long tl = target - __shfl_sync(0xffffffffu, r_prefix, sel_rank);   // target inside this slice
        // one warp per contiguous segment, in index order
        const int seg = (((n + SMP_WARPS - 1) / SMP_WARPS) + 31) & ~31;
        const int s0 = warp * seg, s1 = min(n, s0 + seg);
        unsigned long long wm = 0;
        unsigned wt = 0;
        for (int i = s0 + lane; i < s1; i += 32) {
            const unsigned key = sbuf[i];
            if (key > vstar) wm += key_weight(key);
            else if (key == vstar) ++wt;
        }
        wm = warp_sum_u64(wm);
        wt = (unsigned)warp_sum_u64(wt);
        if (lane == 0) { scratch[warp] = wm; wscan[warp] = wt; }
        __syncthreads();
        if (tid == 0) {
            unsigned long long tb = 0, pre = 0;
            sel_warp = -1;
            for (int w = 0; w < SMP_WARPS; ++w) {
                const unsigned long long kt = my_keep_ties > tb ? min(my_keep_ties - tb, wscan[w]) : 0ull;
                unsigned long long kw = scratch[w] + kt * Wstar;
                if (VERIFY && kept_d && d - lo >= w * seg && d - lo < min(n, w * seg + seg)) kw -= W_d;   // the residual
                if (sel_warp < 0 && tl < pre + kw) { sel_warp = w; sel_prefix = pre; sel_tie_base = tb; }
                pre += kw;
                tb += wscan[w];
            }
        }
        __syncthreads();
        if (warp == sel_warp) {
            unsigned long long run = sel_prefix, tie_rank = sel_tie_base;
            for (int i0 = s0; i0 < s1; i0 += 32) {
                const int i = i0 + lane;
                const unsigned key = i < s1 ? sbuf[i] : 0u;
                const bool tie = i < s1 && key == vstar;
                const unsigned tmask = __ballot_sync(0xffffffffu, tie);
                const unsigned long long my_rank = tie_rank + __popc(tmask & ((1u << lane) - 1u));
                unsigned long long kw = 0;
                if (i < s1 && key > vstar) kw = key_weight(key);
                else if (tie && my_rank < my_keep_ties) kw = Wstar;
                if (VERIFY && lo + i == d) kw = 0;
                const unsigned long long incl = warp_incl_scan_u64(kw, lane);
                const unsigned hit = __ballot_sync(0xffffffffu, kw > 0 && run + incl > tl);
                if (hit) {
                    if (lane == __ffs(hit) - 1) {
                        if constexpr (VERIFY) p.rows[2 * rw] = lo + i;
                        else sample_commit<FILT>(p, b, lo + i);
                    }
                    break;
                }
                run += __shfl_sync(0xffffffffu, incl, 31);
                tie_rank += __popc(tmask);
            }
        }
    }
    cl.sync();   // no CTA leaves while a peer may still read its exchange slots
}

// One thread per request after sample_kernel<true>: k = the first row whose draft was rejected (T - 1 if none), the final token
// from row k, then drop, ids[b, 0], the history, done, the counters and the status bit (row k invalid).  drop = T - the rows that
// stay: k + 1 (the input token and d_1 .. d_k) for a request that goes on; for one that ends in this step (EOS or its limit
// after j appended tokens) only j, the rows of the tokens it emitted before its last one; for one already done none, so its
// caches stay where they ended.  Every request then holds (prompt + emitted tokens - 1) rows.
template <bool FILT>
__device__ void history_append(const SampleParams &p, int b, int token, int lim) {
    int c = p.count[b];
    if (c < lim) {
        p.tokens_out[(size_t)b * p.hist_ld + c] = token;
        p.count[b] = ++c;
        if constexpr (FILT) p.tab[(size_t)b * p.tab_ld + token] += 1u;   // filtered calls count what they append
    }
    bool eos = false;
    for (int k = 0; k < p.n_eos; ++k) eos |= token == p.eos[k];
    if (eos || c >= lim) p.done[b] = 1;
}

template <bool FILT>
__global__ void verify_resolve_kernel(const __grid_constant__ SampleParams p, int B) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int T = p.T;
    const int *row = p.rows + (size_t)b * T * 2;
    int k = 0;
    while (k < T - 1 && (row[2 * k + 1] & ROW_ACCEPT)) ++k;
    const int token = row[2 * k];
    if ((row[2 * k + 1] & ROW_INVALID) && p.status) atomicOr(p.status + (b >> 5), 1 << (b & 31));
    long long *ids = p.ids_out + (size_t)b * p.ids_stride;
    const bool was_done = p.done && p.done[b];
    int keep = was_done ? 0 : k + 1;   // rows of the step that stay: the input token and the accepted drafts
    if (!was_done) {
        if (p.steps) { p.steps[b] += 1; p.accepted[b] += k; }
        if (p.tokens_out) {
            const int lim = (int)min((long long)p.limit[b], p.hist_ld), n0 = p.count[b];
            for (int j = 1; j <= k + 1 && !p.done[b]; ++j) history_append<FILT>(p, b, j <= k ? (int)ids[j] : token, lim);
            // a request that ends here keeps only the rows of the tokens it emitted before its last one
            if (p.done[b]) keep = p.count[b] - n0;
        }
    }
    if (p.drop) p.drop[b] = T - keep;
    ids[0] = token;
}

// Prompt-lookup drafts (mpig_aux_ngram_draft): one cluster of NGR_C CTAs per request.  Every CTA takes the ends e = rank * NGR_THREADS
// + tid + j * NGR_C * NGR_THREADS and keeps the largest (m(e) << 32 | e) with m(e) >= g_min; the CTAs' maxima meet in rank 0, which
// copies the drafts.  A max of integers, so the choice does not depend on the order in which threads finish.
constexpr int NGR_THREADS = 512, NGR_C = 8, NGR_MAX_G = 8, NGR_UNROLL = 4;

__global__ void __launch_bounds__(NGR_THREADS) ngram_draft_kernel(const int *hist, long long ld, const int *len, long long *ids,
                                                                   long long ids_stride, int T, int g_min, int g_max) {
    __shared__ int suf[NGR_MAX_G];
    __shared__ unsigned long long red[NGR_THREADS / 32], best_s;
    cg::cluster_group cl = cg::this_cluster();
    const int rank = (int)cl.block_rank(), b = blockIdx.x / NGR_C, tid = threadIdx.x;
    const int n = (int)min((long long)max(len[b], 0), ld);
    const int *h = hist + (size_t)b * ld;
    if (tid < g_max) suf[tid] = n - 1 - tid >= 0 ? h[n - 1 - tid] : 0;
    __syncthreads();
    unsigned long long best = 0;   // keys with m >= g_min >= 1 are >= 2^32
    if (n >= 2) {
        const int last = suf[0];
        for (int e0 = rank * NGR_THREADS + tid; e0 <= n - 2; e0 += NGR_UNROLL * NGR_C * NGR_THREADS) {
            int v[NGR_UNROLL];
#pragma unroll
            for (int u = 0; u < NGR_UNROLL; ++u) {
                const int e = e0 + u * NGR_C * NGR_THREADS;
                v[u] = e <= n - 2 ? __ldg(h + e) : ~last;
            }
#pragma unroll
            for (int u = 0; u < NGR_UNROLL; ++u) {
                if (v[u] != last) continue;
                const int e = e0 + u * NGR_C * NGR_THREADS;
                int m = 1;
                while (m < g_max && e - m >= 0 && __ldg(h + e - m) == suf[m]) ++m;
                if (m >= g_min) best = max(best, (unsigned long long)m << 32 | (unsigned)e);
            }
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if ((tid & 31) == 0) red[tid >> 5] = best;
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < NGR_THREADS / 32; ++w) best = max(best, red[w]);
        best_s = best;
    }
    cl.sync();
    if (rank == 0 && tid == 0) {
        for (int r = 1; r < NGR_C; ++r) best = max(best, *cl.map_shared_rank(&best_s, r));
        long long *out = ids + (size_t)b * ids_stride;
        for (int i = 0; i < T - 1; ++i) {
            long long tok;
            if (best == 0) tok = n >= 1 ? h[n - 1] : 0;
            else {
                const int j = (int)(best & 0xffffffffu) + 1 + i;   // h' = h followed by the drafts: an overlapping copy
                tok = j < n ? h[j] : out[1 + j - n];
            }
            out[1 + i] = tok;
        }
    }
    cl.sync();   // rank 0 reads every peer's best_s
}

}  // namespace mpig

using namespace mpig;

namespace {

// cluster size and slice of a row of V logits; false when V is beyond what SMP_MAX_C CTAs' shared memory holds
bool sample_layout(int V, int &C, int &slice) {
    C = std::min(SMP_MAX_C, (V + SMP_ROWS_PER_CTA_HINT - 1) / SMP_ROWS_PER_CTA_HINT);
    slice = ((V + C - 1) / C + SMP_SLICE_ALIGN - 1) / SMP_SLICE_ALIGN * SMP_SLICE_ALIGN;
    return (size_t)slice * 4 <= (size_t)SMP_SMEM_CAP;
}

int check_filters(const mpig_sample_filters *f, int V, const char *fn) {
    MPIG_REQUIRE(f, MPIG_EINVAL, "%s: filters is null", fn);
    MPIG_REQUIRE(f->top_k && f->min_p && f->repetition_penalty && f->presence_penalty && f->frequency_penalty && f->table,
                 MPIG_EINVAL, "%s: every filter array and the table are required", fn);
    const void *aligned4[] = {f->top_k, f->min_p, f->repetition_penalty, f->presence_penalty, f->frequency_penalty, f->table};
    for (const void *q : aligned4)
        MPIG_REQUIRE(((uintptr_t)q & 3) == 0, MPIG_EINVAL, "%s: misaligned filter array or table", fn);
    MPIG_REQUIRE(f->ld >= V, MPIG_EINVAL, "%s: table ld=%lld < V=%d", fn, (long long)f->ld, V);
    return MPIG_OK;
}

void set_filters(SampleParams &prm, const mpig_sample_filters *f) {
    if (!f) return;
    prm.top_k = f->top_k; prm.min_p = f->min_p; prm.rep = f->repetition_penalty; prm.pres = f->presence_penalty;
    prm.freq = f->frequency_penalty; prm.tab = f->table; prm.tab_ld = f->ld;
}

template <bool VERIFY, bool FILT>
int launch_rows(const SampleParams &prm, int rows, cudaStream_t stream) {
    MPIG_FUNC_ATTR((sample_kernel<VERIFY, FILT>), cudaFuncAttributeMaxDynamicSharedMemorySize, SMP_SMEM_CAP);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(rows * prm.C);
    cfg.blockDim = dim3(SMP_THREADS);
    cfg.dynamicSmemBytes = (size_t)prm.slice * 4;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = prm.C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    MPIG_CUDA(cudaLaunchKernelEx(&cfg, sample_kernel<VERIFY, FILT>, prm));
    return MPIG_OK;
}

int sample_impl(const char *fn, const float *logits, int B, int V, int64_t ld, const float *temperature, const float *top_p,
                uint64_t seed, const uint64_t *offset, int64_t *ids_out, int64_t ids_stride, int32_t *tokens_out, int32_t *count,
                int32_t *done, int max_new, const int32_t *eos_ids, int n_eos, int32_t *status, int64_t *debug, float *debug_w,
                const mpig_sample_filters *filters, void *stream) {
    MPIG_REQUIRE(B >= 1 && V >= 1, MPIG_EINVAL, "%s: B=%d and V=%d must be >= 1", fn, B, V);
    int C, slice;
    MPIG_REQUIRE(sample_layout(V, C, slice), MPIG_EINVAL, "%s: V=%d exceeds what %d CTAs' shared memory holds (%d)", fn, V,
                 SMP_MAX_C, SMP_MAX_C * (SMP_SMEM_CAP / 4));
    MPIG_REQUIRE(ld >= V, MPIG_EINVAL, "%s: ld=%lld < V=%d", fn, (long long)ld, V);
    MPIG_REQUIRE(logits && ((uintptr_t)logits & 3) == 0, MPIG_EINVAL, "%s: logits null or misaligned", fn);
    MPIG_REQUIRE(temperature && top_p && offset, MPIG_EINVAL, "%s: temperature, top_p and offset are required", fn);
    MPIG_REQUIRE(((uintptr_t)temperature & 3) == 0 && ((uintptr_t)top_p & 3) == 0 && ((uintptr_t)offset & 7) == 0, MPIG_EINVAL,
                 "%s: misaligned temperature, top_p or offset", fn);
    MPIG_REQUIRE(n_eos >= 0 && n_eos <= SMP_MAX_EOS && (n_eos == 0 || eos_ids), MPIG_EINVAL,
                 "%s: n_eos=%d outside [0, %d] (or eos_ids null)", fn, n_eos, SMP_MAX_EOS);
    MPIG_REQUIRE(!tokens_out || (count && done && max_new >= 1), MPIG_EINVAL, "%s: tokens_out needs count, done and max_new >= 1", fn);
    MPIG_REQUIRE(!ids_out || ids_stride >= 1, MPIG_EINVAL, "%s: ids_stride=%lld < 1", fn, (long long)ids_stride);
    MPIG_REQUIRE((long long)B * C <= INT_MAX, MPIG_EINVAL, "%s: B=%d too large", fn, B);

    SampleParams prm = {};
    prm.logits = logits; prm.ld = ld; prm.V = V; prm.C = C; prm.slice = slice;
    prm.temperature = temperature; prm.top_p = top_p; prm.seed = seed; prm.offset = (const unsigned long long *)offset;
    prm.ids_out = (long long *)ids_out; prm.ids_stride = ids_stride;
    prm.tokens_out = tokens_out; prm.count = count; prm.done = done; prm.max_new = max_new;
    prm.n_eos = n_eos;
    for (int i = 0; i < n_eos; ++i) prm.eos[i] = eos_ids[i];
    prm.status = status; prm.dbg = (long long *)debug; prm.dbg_w = debug_w;
    prm.T = 1;
    set_filters(prm, filters);
    return filters ? launch_rows<false, true>(prm, B, as_stream(stream)) : launch_rows<false, false>(prm, B, as_stream(stream));
}

int verify_impl(const char *fn, const float *logits, int B, int T, int V, int64_t ld_b, int64_t ld_t, const float *temperature,
                const float *top_p, uint64_t seed, const uint64_t *offset, int64_t *ids, int64_t ids_stride, int32_t *rows,
                int32_t *drop, int32_t *history, int64_t history_ld, int32_t *length, const int32_t *limit, int32_t *done,
                int32_t *steps, int32_t *accepted, const int32_t *eos_ids, int n_eos, int32_t *status, int64_t *debug,
                float *debug_w, const mpig_sample_filters *filters, void *stream) {
    MPIG_REQUIRE(B >= 1 && V >= 1, MPIG_EINVAL, "%s: B=%d and V=%d must be >= 1", fn, B, V);
    MPIG_REQUIRE(T >= 1 && T <= SMP_MAX_VERIFY_T, MPIG_EINVAL, "%s: T=%d outside [1, %d]", fn, T, SMP_MAX_VERIFY_T);
    int C, slice;
    MPIG_REQUIRE(sample_layout(V, C, slice), MPIG_EINVAL, "%s: V=%d exceeds what %d CTAs' shared memory holds (%d)", fn, V,
                 SMP_MAX_C, SMP_MAX_C * (SMP_SMEM_CAP / 4));
    MPIG_REQUIRE(ld_t >= V && ld_b >= (T - 1) * ld_t + V, MPIG_EINVAL, "%s: strides ld_b=%lld, ld_t=%lld overlap rows of V=%d", fn,
                 (long long)ld_b, (long long)ld_t, V);
    MPIG_REQUIRE(logits && ((uintptr_t)logits & 3) == 0, MPIG_EINVAL, "%s: logits null or misaligned", fn);
    MPIG_REQUIRE(temperature && top_p && offset, MPIG_EINVAL, "%s: temperature, top_p and offset are required", fn);
    MPIG_REQUIRE(((uintptr_t)temperature & 3) == 0 && ((uintptr_t)top_p & 3) == 0 && ((uintptr_t)offset & 7) == 0, MPIG_EINVAL,
                 "%s: misaligned temperature, top_p or offset", fn);
    MPIG_REQUIRE(ids && ((uintptr_t)ids & 7) == 0 && ids_stride >= T, MPIG_EINVAL, "%s: ids null, misaligned or ids_stride=%lld < T=%d",
                 fn, (long long)ids_stride, T);
    MPIG_REQUIRE(rows && ((uintptr_t)rows & 3) == 0, MPIG_EINVAL, "%s: rows (B, T, 2) null or misaligned", fn);
    MPIG_REQUIRE(n_eos >= 0 && n_eos <= SMP_MAX_EOS && (n_eos == 0 || eos_ids), MPIG_EINVAL,
                 "%s: n_eos=%d outside [0, %d] (or eos_ids null)", fn, n_eos, SMP_MAX_EOS);
    MPIG_REQUIRE(!history || (length && limit && done && history_ld >= 1), MPIG_EINVAL,
                 "%s: history needs length, limit, done and history_ld >= 1", fn);
    MPIG_REQUIRE(!steps == !accepted, MPIG_EINVAL, "%s: steps and accepted go together", fn);
    const void *aligned4[] = {drop, history, length, limit, done, steps, accepted, status, debug_w};
    for (const void *q : aligned4) MPIG_REQUIRE(((uintptr_t)q & 3) == 0, MPIG_EINVAL, "%s: misaligned int32 / fp32 argument", fn);
    MPIG_REQUIRE(((uintptr_t)debug & 7) == 0, MPIG_EINVAL, "%s: misaligned debug", fn);
    MPIG_REQUIRE((long long)B * T * C <= INT_MAX, MPIG_EINVAL, "%s: B=%d too large", fn, B);

    SampleParams prm = {};
    prm.logits = logits; prm.ld = ld_b; prm.ld_t = ld_t; prm.V = V; prm.C = C; prm.slice = slice; prm.T = T;
    prm.temperature = temperature; prm.top_p = top_p; prm.seed = seed; prm.offset = (const unsigned long long *)offset;
    prm.ids_out = (long long *)ids; prm.ids_stride = ids_stride; prm.rows = rows; prm.drop = drop;
    prm.tokens_out = history; prm.hist_ld = history_ld; prm.count = length; prm.limit = const_cast<int *>(limit); prm.done = done;
    prm.steps = steps; prm.accepted = accepted;
    prm.n_eos = n_eos;
    for (int i = 0; i < n_eos; ++i) prm.eos[i] = eos_ids[i];
    prm.status = status; prm.dbg = (long long *)debug; prm.dbg_w = debug_w;
    set_filters(prm, filters);

    const cudaStream_t st = as_stream(stream);
    const int rc = filters ? launch_rows<true, true>(prm, B * T, st) : launch_rows<true, false>(prm, B * T, st);
    if (rc != MPIG_OK) return rc;
    if (filters) verify_resolve_kernel<true><<<(B + 127) / 128, 128, 0, st>>>(prm, B);
    else verify_resolve_kernel<false><<<(B + 127) / 128, 128, 0, st>>>(prm, B);
    MPIG_CUDA(cudaGetLastError());
    return MPIG_OK;
}

}  // namespace

extern "C" {

int mpig_aux_sample(const float *logits, int B, int V, int64_t ld, const float *temperature, const float *top_p, uint64_t seed,
                    const uint64_t *offset, int64_t *ids_out, int64_t ids_stride, int32_t *tokens_out, int32_t *count,
                    int32_t *done, int max_new, const int32_t *eos_ids, int n_eos, int32_t *status, int64_t *debug,
                    float *debug_w, void *stream) {
    return sample_impl("mpig_aux_sample", logits, B, V, ld, temperature, top_p, seed, offset, ids_out, ids_stride, tokens_out, count,
                       done, max_new, eos_ids, n_eos, status, debug, debug_w, nullptr, stream);
}

int mpig_aux_sample_filtered(const float *logits, int B, int V, int64_t ld, const float *temperature, const float *top_p,
                             uint64_t seed, const uint64_t *offset, int64_t *ids_out, int64_t ids_stride, int32_t *tokens_out,
                             int32_t *count, int32_t *done, int max_new, const int32_t *eos_ids, int n_eos, int32_t *status,
                             int64_t *debug, float *debug_w, const mpig_sample_filters *filters, void *stream) {
    const int rc = check_filters(filters, V, "mpig_aux_sample_filtered");
    if (rc != MPIG_OK) return rc;
    return sample_impl("mpig_aux_sample_filtered", logits, B, V, ld, temperature, top_p, seed, offset, ids_out, ids_stride, tokens_out,
                       count, done, max_new, eos_ids, n_eos, status, debug, debug_w, filters, stream);
}

int mpig_aux_sample_occupancy(int V, int *clusters) {
    MPIG_REQUIRE(V >= 1 && clusters, MPIG_EINVAL, "mpig_aux_sample_occupancy: bad arguments");
    int C, slice;
    MPIG_REQUIRE(sample_layout(V, C, slice), MPIG_EINVAL, "mpig_aux_sample_occupancy: V=%d too large", V);
    MPIG_FUNC_ATTR((sample_kernel<false, false>), cudaFuncAttributeMaxDynamicSharedMemorySize, SMP_SMEM_CAP);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(C);
    cfg.blockDim = dim3(SMP_THREADS);
    cfg.dynamicSmemBytes = (size_t)slice * 4;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    MPIG_CUDA(cudaOccupancyMaxActiveClusters(clusters, (const void *)sample_kernel<false, false>, &cfg));
    return MPIG_OK;
}

int mpig_aux_verify_sample(const float *logits, int B, int T, int V, int64_t ld_b, int64_t ld_t, const float *temperature,
                           const float *top_p, uint64_t seed, const uint64_t *offset, int64_t *ids, int64_t ids_stride,
                           int32_t *rows, int32_t *drop, int32_t *history, int64_t history_ld, int32_t *length, const int32_t *limit,
                           int32_t *done, int32_t *steps, int32_t *accepted, const int32_t *eos_ids, int n_eos, int32_t *status,
                           int64_t *debug, float *debug_w, void *stream) {
    return verify_impl("mpig_aux_verify_sample", logits, B, T, V, ld_b, ld_t, temperature, top_p, seed, offset, ids, ids_stride, rows,
                       drop, history, history_ld, length, limit, done, steps, accepted, eos_ids, n_eos, status, debug, debug_w,
                       nullptr, stream);
}

int mpig_aux_verify_sample_filtered(const float *logits, int B, int T, int V, int64_t ld_b, int64_t ld_t, const float *temperature,
                                    const float *top_p, uint64_t seed, const uint64_t *offset, int64_t *ids, int64_t ids_stride,
                                    int32_t *rows, int32_t *drop, int32_t *history, int64_t history_ld, int32_t *length,
                                    const int32_t *limit, int32_t *done, int32_t *steps, int32_t *accepted, const int32_t *eos_ids,
                                    int n_eos, int32_t *status, int64_t *debug, float *debug_w, const mpig_sample_filters *filters,
                                    void *stream) {
    const int rc = check_filters(filters, V, "mpig_aux_verify_sample_filtered");
    if (rc != MPIG_OK) return rc;
    return verify_impl("mpig_aux_verify_sample_filtered", logits, B, T, V, ld_b, ld_t, temperature, top_p, seed, offset, ids,
                       ids_stride, rows, drop, history, history_ld, length, limit, done, steps, accepted, eos_ids, n_eos, status, debug,
                       debug_w, filters, stream);
}

int mpig_aux_ngram_draft(const int32_t *history, int B, int64_t ld, const int32_t *length, int64_t *ids, int64_t ids_stride, int T,
                         int g_min, int g_max, void *stream) {
    MPIG_REQUIRE(B >= 1 && ld >= 1, MPIG_EINVAL, "mpig_aux_ngram_draft: B=%d and ld=%lld must be >= 1", B, (long long)ld);
    MPIG_REQUIRE(ld <= INT_MAX, MPIG_EINVAL, "mpig_aux_ngram_draft: ld=%lld too large", (long long)ld);
    MPIG_REQUIRE(T >= 1 && T <= SMP_MAX_VERIFY_T, MPIG_EINVAL, "mpig_aux_ngram_draft: T=%d outside [1, %d]", T, SMP_MAX_VERIFY_T);
    MPIG_REQUIRE(g_min >= 1 && g_min <= g_max && g_max <= NGR_MAX_G, MPIG_EINVAL,
                 "mpig_aux_ngram_draft: need 1 <= g_min=%d <= g_max=%d <= %d", g_min, g_max, NGR_MAX_G);
    MPIG_REQUIRE(history && length && ids, MPIG_EINVAL, "mpig_aux_ngram_draft: history, length and ids are required");
    MPIG_REQUIRE(((uintptr_t)history & 3) == 0 && ((uintptr_t)length & 3) == 0 && ((uintptr_t)ids & 7) == 0, MPIG_EINVAL,
                 "mpig_aux_ngram_draft: misaligned history, length or ids");
    MPIG_REQUIRE(ids_stride >= T, MPIG_EINVAL, "mpig_aux_ngram_draft: ids_stride=%lld < T=%d", (long long)ids_stride, T);
    MPIG_REQUIRE((long long)B * NGR_C <= INT_MAX, MPIG_EINVAL, "mpig_aux_ngram_draft: B=%d too large", B);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(B * NGR_C);
    cfg.blockDim = dim3(NGR_THREADS);
    cfg.stream = as_stream(stream);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = NGR_C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    MPIG_CUDA(cudaLaunchKernelEx(&cfg, ngram_draft_kernel, (const int *)history, (long long)ld, (const int *)length, (long long *)ids,
                                 (long long)ids_stride, T, g_min, g_max));
    return MPIG_OK;
}

}  // extern "C"
