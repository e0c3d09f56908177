// common.cuh -- context layout, error plumbing and PTX wrappers shared by the sm_90a kernels.
//
// HBM layout owned by a context (all per SPARSE layer unless noted; B requests, C context slots (mpig_config.num_contexts, 0 = B),
// Hkv kv-heads, M = max_length rows of capacity, d = head_dim, REC = 2*d bf16 = 512 B at d = 128).  The sampled store and the
// tables are per SLOT; request b reads slot slot_of[b] (slot group slot_of[b]*Hkv + h/G), its window and lengths are its own:
//
//   kv      [C][Hkv][M]      REC-byte records  { K row (d bf16) | V row (d bf16) }   one index -> one burst
//   kn      [C][Hkv][M]      fp32 key norms (as given to fill; reference sparse_attention.h:45)
//   offsets [C][Hkv][L][S][NB+1] int32 per-segment CSR bucket starts, absolute positions in the table's item row
//                            (replaces table_start/table_end, lsh.h:38-39); S = nseg equal key segments of seg_len <= 65536
//                            keys, sized to the probing cluster (DESIGN.md section 2)
//   items   [C][Hkv][L][M]   uint16 key index - seg_len * segment, segment-major, then grouped by bucket (lsh.h:40 keeps int32)
//   win     [B][Hkv][Wcap]   REC-byte records of the sink+local+generated window (keys centred)
//   avg_k   [B][Hkv][d]      bf16 mean offloaded key (attnserver.py:142-148)
//   dense   [B][Hkv][M]      REC-byte records (dense layers, only with alloc_dense_kv)
//
// Shared dense mode (mpig_config.dense_tail_rows = R > 0, only with C < B): per dense layer the prompt rows live once per
// slot and the rows a request adds after its prompt in a tail of its own.  Row r of request b is row r of slot slot_of[b]'s store
// when r < dense_base[b], else row r - dense_base[b] of b's tail:
//   dense   [C][Hkv][M]      REC-byte records (the slot store)
//   tail    [B][Hkv][R]      REC-byte records (the request tail)
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/magicpig_b200.h"

namespace mpig {

void set_error(const char *fmt, ...);

#define MPIG_CUDA(call)                                                                          \
    do {                                                                                         \
        cudaError_t _e = (call);                                                                 \
        if (_e != cudaSuccess) {                                                                 \
            ::mpig::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
            return MPIG_ECUDA;                                                                   \
        }                                                                                        \
    } while (0)

#define MPIG_REQUIRE(cond, code, ...)        \
    do {                                     \
        if (!(cond)) {                       \
            ::mpig::set_error(__VA_ARGS__);  \
            return (code);                   \
        }                                    \
    } while (0)

#define MPIG_LAUNCH_CHECK(ctx)                \
    do {                                      \
        (ctx)->launches++;                    \
        MPIG_CUDA(cudaGetLastError());        \
    } while (0)

// cudaFuncSetAttribute is per DEVICE: remembered per (function, attribute, current device, value), thread-safe (context.cu)
int func_attr_once(const void *fn, cudaFuncAttribute attr, int value);
#define MPIG_FUNC_ATTR(fn, attr, value)                                        \
    do {                                                                       \
        int _rc = ::mpig::func_attr_once((const void *)(fn), (attr), (value)); \
        if (_rc != MPIG_OK) return _rc;                                        \
    } while (0)

constexpr int TREE_MAX = 8;        // nodes of a verification step (mpig_reserve_query_tokens caps t_max at this)

// step_buf views (see mpig_ctx::step_buf): ancestor masks, parents, step bases; T = the pending step's node count
template <typename I> __host__ __device__ inline I *step_masks(I *buf) { return buf; }
template <typename I> __host__ __device__ inline I *step_parents(I *buf, int B) { return buf + (size_t)B * TREE_MAX; }
template <typename I> __host__ __device__ inline I *step_bases(I *buf, int B) { return buf + (size_t)2 * B * TREE_MAX; }

constexpr int SEG_BITS = 16;      // table items are uint16 offsets inside key segments of at most 2^16 keys (tables.cu)
constexpr int SEG = 1 << SEG_BITS;

struct LayerStore {
    bool sparse = false;
    bool dense = false;
    uint8_t *kv = nullptr;       // sparse: offloaded records
    float *kn = nullptr;
    int32_t *offsets = nullptr;
    int32_t *items = nullptr;    // storage of the uint16 item rows [C*Hkv][L][M]
    uint8_t *win = nullptr;      // window records
    __nv_bfloat16 *avg_k = nullptr;
    uint8_t *dense_kv = nullptr; // dense: full-context records ([B][Hkv][M]), or the slot store ([C][Hkv][M]) in shared dense mode
    uint8_t *dense_tail = nullptr; // dense, shared dense mode only: the request tails [B][Hkv][R]
};

// one entry of the accept kernel's layer table: the REC-byte rows of a sparse window ([BG][cap], cap = Wcap) or of a dense KV
// cache ([BG][cap], cap = max_length, or the request tails with cap = R in shared dense mode); dense = 1 selects dense_len and the
// dense step base.  The reorder kernel walks the same table: a sparse entry also carries the layer's avg_k ([BG][d], null for a
// dense entry), and x0 is the entry's first CTA column in the reorder grid (Hkv * ceil(cap / REORDER_ROWS) columns per entry).
struct AcceptLayer {
    uint8_t *rows;
    int cap;
    int dense;
    __nv_bfloat16 *avg_k;
    int x0;
};
constexpr int REORDER_ROWS = 64;   // rows one CTA of the reorder kernel copies (32 KB of records)

struct AttendTuning {
    int ctas = 0;    // 0 = one per SM * occupancy
    int warps = 12;
    int tma = 1;     // 1 = per-row cp.async.bulk (TMA engine), 0 = per-row 32 x 16 B cp.async (LSU path)
};

// The verification step between a plan and its rewind or accept.  Only begin() and end() write it: the plans begin a step
// (step.cu); rewind and accept end it, and so do mpig_clear, mpig_fork_request, mpig_bind_request and mpig_reorder_requests.
struct PendingStep {
    int T = 0;            // node count of the last plan (0 = no plan since create / clear); decode_tokens must match it
    bool open = false;    // the step may still be rewound or accepted (at most once per plan)
    bool tree = false;    // the step came from mpig_plan_tree (mpig_rewind is refused)
    bool chunk = false;   // the step came from mpig_plan_chunk (only mpig_chunk_attend decodes it; mpig_accept is refused)
    void begin(int t, bool is_tree, bool is_chunk = false) {
        T = t;
        open = true;
        tree = is_tree;
        chunk = is_chunk;
    }
    // forget = true (mpig_clear): no step to decode either
    void end(bool forget = false) {
        open = false;
        if (forget) {
            T = 0;
            tree = false;
            chunk = false;
        }
    }
};

}  // namespace mpig

struct mpig_peer;

struct mpig_ctx {
    mpig_config cfg;
    int nseg = 1;      // key segments per table row: ceil(M / 65536) (tables.cu)
    int seg_len = 0;   // keys per segment: ceil(M / nseg) rounded up to 64 -- equal segments, so a probing cluster's CTAs own equal ranges
    int NB = 0, Wcap = 0, G = 0, H = 0 /* B*Hq */, BG = 0 /* B*Hkv */, rec_bytes = 0, num_sms = 0;
    int bitmap_words = 0;  // ceil(M/32)
    int cta_per_sm = 1;    // probing / fused CTAs per SM the geometry is planned for (mpig_config.ctas_per_sm == 2 -> 2)
    int max_cluster = 8;   // largest probing / fused cluster whose B*Hq copies are all resident at once (mpig_create)
    std::vector<mpig::LayerStore> layers;
    std::vector<std::vector<int>> n_off;  // [layer][slot] offloaded key count (host bookkeeping)
    // context slots: the sampled store and the tables exist once per slot, request b reads slot slot_of[b].  The device map is
    // allocated at create time and never moves (a captured step reads the bindings of the replay); h_slot_of mirrors it.  Only
    // copy-engine calls write it, never a kernel: mpig_clear, mpig_fork_request and mpig_bind_request upload it, and
    // mpig_reorder_requests has its kernel write the new map into slot_stage and then copies that into slot_of with a
    // device-to-device memcpy (a memcpy node under capture).  So the decode kernels may read it before griddepcontrol.wait.
    int C = 0;                            // number of slots (1..B)
    int32_t *slot_of = nullptr;           // [B]
    int32_t *slot_stage = nullptr;        // [B] the reorder kernel's new map, copied into slot_of after it
    std::vector<int> h_slot_of;           // [B]
    // h_slot_of and h_dense_base equal the device maps unless a reorder was captured into a CUDA graph (its replays change only
    // the device maps): while false, every host path that reads them refreshes them first (refresh_maps).  mpig_clear sets it
    // again, unless a reorder has ever been captured: that graph may be replayed after the clear.
    bool h_map_exact = true;
    bool reorder_captured = false;
    // the map the kernels get: null while every request owns its slot (C = B, bindings fixed), so that path addresses b itself
    const int32_t *slot_map() const { return C < cfg.batch_size ? slot_of : nullptr; }
    // shared dense mode (R = dense_tail_rows > 0): the prompt rows of the dense layers live once per slot, each request's later
    // rows in its own tail of R rows.  dense_base[b] = the first row of request b that lies in its tail (set by mpig_dense_fill,
    // mpig_fork_request and the reorder kernel, zeroed by mpig_clear); allocated at create time and never moved, h_dense_base
    // mirrors it (exactly while h_map_exact).  The decode kernels read it only after griddepcontrol.wait.
    int dense_tail_rows = 0;
    int32_t *dense_base = nullptr;        // [B], shared dense mode only
    std::vector<int> h_dense_base;        // [B]
    // the base map the kernels get: null in the default layout
    const int32_t *dense_base_map() const { return dense_tail_rows > 0 ? dense_base : nullptr; }
    // the dense capacity of request b: max_length, or min(max_length, base + R) in shared dense mode.  Read only by the plans'
    // host-mirror checks, which run only while h_len_exact; a captured reorder clears h_len_exact with h_map_exact and only
    // mpig_clear sets both again, so h_dense_base is exact wherever this is read.
    int dense_cap(int b) const {
        return dense_tail_rows > 0 ? std::min(cfg.max_length, h_dense_base[b] + dense_tail_rows) : cfg.max_length;
    }
    // shared spill mode (mpig_config.shared_spill = 1, DESIGN.md section 3.12): requests that share a slot spill into it, and each
    // spilled key is private.  Keys [private_lo[layer][slot], ...) of a slot's store are private; the private key at offset p is
    // seen by request b iff bit b of vis[slot][p] is set.  Both arrays are allocated at create time and never move (a captured
    // step reads the current ones).  Kernels write them (fills, spill, fork, bind) as well as mpig_clear's memsets, so the decode
    // kernels read them only after griddepcontrol.wait.
    bool shared_spill = false;
    uint32_t *vis = nullptr;              // [C][max_length]
    int32_t *private_lo = nullptr;        // [num_layers][C]
    std::vector<std::vector<int>> h_private_lo;   // [layer][slot], mirrors private_lo
    // the maps the kernels get: null unless in shared spill mode
    const uint32_t *vis_map() const { return shared_spill ? vis : nullptr; }
    const int32_t *private_lo_map(int layer) const { return shared_spill ? private_lo + (size_t)layer * C : nullptr; }
    // global state
    __nv_bfloat16 *hash_func = nullptr;   // (d, K*L) as given
    __nv_bfloat16 *hash_func_t = nullptr; // (K*L, d) transposed copy: K-major B operand for the SimHash GEMM
    int32_t *win_len = nullptr;           // [B] current window length (sink+local+generated so far)
    int32_t *dense_len = nullptr;         // [B]
    // per-step scratch (decode is allocation-free)
    int32_t *codes = nullptr;             // [H][L]
    float *qnorm = nullptr;               // [H]
    int32_t *results = nullptr;           // [H][M]
    int32_t *nnz = nullptr;               // [H]
    uint32_t *bitmaps = nullptr;          // [H][2][bitmap_words]  (only written when save_mask)
    float *partials = nullptr;            // stream-K partial states
    int32_t *counters = nullptr;          // [H] merge tickets (self-resetting)
    float *mve = nullptr;                 // [2][H]
    void *host_stage = nullptr;           // pinned staging for *_host calls
    void *dev_stage = nullptr;            // device staging for *_host calls
    size_t bytes = 0;
    uint64_t launches = 0;
    int save_mask = 0;
    int max_partial_warps = 0;
    mpig::AttendTuning attend;
    unsigned long long *dbg_buf = nullptr;   // attend stage timestamps when option "attend_debug" is set
    int attend_debug = 0;
    int attend_skip = 0;
    int dense_impl = 1;  // 1 = GQA-shared dense kernel (attend_dense.cu), 0 = the gather kernel (attend_mma.cu) in range mode
    bool hash_func_set = false;  // mpig_set_hash_func has been called (hashing with the zero projection is refused)
    int pdl_first = 1;     // launch the first kernel of a decode (simhash) with programmatic stream serialization as well
    int keyhash_skip = 0;  // debug/timing only: 1 = no stores, 2 = no sign pack, 4 = no MMAs (results are wrong)
    int keyhash_impl = 1;  // 1 = persistent warp-specialised pipeline (keyhash.cu), 0 = one tile per CTA
    std::vector<cudaEvent_t> timing_events;  // 4 per timed decode call
    int timing_calls = 0;
    // decode variant: 1 = ONE fused launch per sparse layer (fused.cu) wherever its shape rules allow, 0 = three launches
    int decode_impl = 1;
    int fused_selcap = 2048;                 // selected keys a CTA of the fused kernel lists per pass (shared-memory list)
    int fused_kreg = 0;                      // 1 = K halves of the rows go HBM -> registers, V halves TMA -> shared memory; 0 = whole records by TMA
    int fused_debug = 0;                     // record per-CTA phase clocks of the fused kernel into fused_dbg
    unsigned long long *fused_dbg = nullptr; // [max CTAs][16]
    int fused_issue_win = 8;                 // warps of a fused-kernel CTA that issue row requests at the same time (fused.cu, P5); 0 = all
    void *fused_plan_cache = nullptr;        // fused.cu: the launch plans (geometry, shared-memory carve-up) for T = 1..8 tokens
    long long fused_plan_key[9] = {0};       //   ... and the option values each was computed for
    int last_decode_fused = 0;               // which variant the last mpig_decode ran (mpig_get_info)
    // fp32 copy of the attention output before the ABI's bf16 rounding (option "out_f32"; parity tests apply the 1e-3 bar here)
    int want_out_f32 = 0;
    float *out_f32 = nullptr;                // [H][d]
    // capacity bookkeeping (the window / the dense cache saturate silently on the device): a device flag raised by
    // plan_kernel plus a host mirror that is exact as long as plan() is not replayed from a CUDA graph
    int32_t *err_flag = nullptr;             // bits: see mpig_error_flags (0 window full, 1 dense full, 2 rewind, 3 tree, 4 reorder)
    std::vector<int> h_win_len, h_dense_len; // [B]
    bool h_len_exact = true;
    void *host_stage_dev = nullptr;          // device-side address of the mapped pinned block host_stage
    uint32_t host_epoch = 0;                 // completion-flag value of the last mpig_decode_host (flags live at the end of host_stage)
    // mpig_spill_window scratch, allocated by the first spill: per-request counts | spilled keys (Hkv, g, d) bf16 per request |
    // their codes (Hkv, L, g) int16 per request, sized for every request spilling all its non-sink window rows
    uint8_t *spill_buf = nullptr;
    // multi-token verification steps (mpig_reserve_query_tokens / mpig_plan_tokens / mpig_decode_tokens / mpig_rewind).  After the
    // reservation the per-step scratch above (codes, qnorm, results, nnz, bitmaps, mve, out_f32) holds B*tok_max*Hq rows.
    int tok_max = 1;                         // largest T a step may verify (1 until mpig_reserve_query_tokens)
    mpig::PendingStep pending;               // the step of the last plan (step.cu)
    int last_tokens = 1;                     // rows of the readers (mpig_last_probe / _codes / _out_f32) = B * last_tokens * Hq
    bool last_chunk = false;                 // the last attention call was a chunk step: it has no probe or codes to read
    bool plan_captured = false;              // a plan has been captured into a CUDA graph (the scratch addresses are baked in)
    int last_tokens_waves = 0;               // cluster waves of the last mpig_decode_tokens launch
    int last_chunk_splits = 0;               // key splits of the last mpig_chunk_attend launch (0 before any)
    // token trees (mpig_plan_tree / mpig_accept).  step_buf is allocated at create time for the largest step (8 nodes), so it never
    // moves: int32 [B][T] ancestor masks (bit j of node t = node j is t or one of its ancestors) | int32 [B][T] parents | int32
    // [B][2] step bases (window, dense length before the plan, after saturation).  Every plan writes it (chains for plan_tokens).
    int32_t *step_buf = nullptr;
    // device table of the layers that own rows (sparse windows and dense KV), for the one-launch accept and reorder kernels
    void *accept_layers = nullptr;
    int n_accept_layers = 0;
    int reorder_cols = 0;                    // CTA columns of the reorder kernel's copy grid (the last entry's x0 + its columns)
    // chunk steps (mpig_reserve_chunk_tokens / mpig_plan_chunk / mpig_chunk_attend, attend_chunk.cu).  store_n mirrors n_off on the
    // device ([num_layers][C], written by the fills, the spill and mpig_clear) so that a captured chunk step reads the store length
    // of the replay.  The split scratch is allocated by the reservation and never moves after a capture.
    int chunk_max = 0;                       // largest T of a chunk step (0 until mpig_reserve_chunk_tokens)
    int32_t *store_n = nullptr;              // [num_layers][C]
    float *chunk_partials = nullptr;         // [chunk_part_tiles][CK_ROWS][PART_FLOATS] split states
    int32_t *chunk_counters = nullptr;       // [B*Hkv][m-blocks of t_max] merge tickets (self-resetting)
    int chunk_part_tiles = 0;
};

namespace mpig {

// Every entry point runs on the context's device and leaves the caller's current device as it found it.
struct DeviceGuard {
    int prev = -1;
    bool switched = false;
    explicit DeviceGuard(const mpig_ctx *ctx) {
        if (!ctx) return;
        if (cudaGetDevice(&prev) == cudaSuccess && prev != ctx->cfg.device) switched = (cudaSetDevice(ctx->cfg.device) == cudaSuccess);
    }
    ~DeviceGuard() {
        if (switched) cudaSetDevice(prev);
    }
    DeviceGuard(const DeviceGuard &) = delete;
    DeviceGuard &operator=(const DeviceGuard &) = delete;
};

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float bf16_bits_to_f32(uint32_t lo16) { return __uint_as_float(lo16 << 16); }
// low / high bf16 of a packed pair
__device__ __forceinline__ float bf16lo(uint32_t p) { return __uint_as_float(p << 16); }
__device__ __forceinline__ float bf16hi(uint32_t p) { return __uint_as_float(p & 0xffff0000u); }

// FBGEMM's fp32->bf16 (FbgemmBfloat16ConvertAvx512.cc:20-26): add 2^15, truncate.  NaN kept NaN.
__device__ __forceinline__ uint16_t f32_to_bf16_half_up(float f) {
    uint32_t u = __float_as_uint(f);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40u);
    return (uint16_t)((u + 0x8000u) >> 16);
}
// torch's bf16 rounding (RNE)
__device__ __forceinline__ uint16_t f32_to_bf16_rne(float f) {
    return __bfloat16_as_ushort(__float2bfloat16_rn(f));
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier + 1-D bulk async copy (TMA engine; SASS: UBLKCP, SYNCS) -----------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    // relaxed: nothing this thread wrote earlier has to be published by the arrive (the default .release made the
    // first arrive of every warp wait ~4.7 us for the thread's outstanding memory operations)
    asm volatile("mbarrier.arrive.expect_tx.relaxed.cta.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// plain arrive (count 1), relaxed for the same reason
__device__ __forceinline__ void mbar_arrive_relaxed(uint64_t *bar) {
    asm volatile("mbarrier.arrive.relaxed.cta.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// global -> shared bulk copy, completion counted in bytes on `bar`.  16-B aligned src/dst, size % 16 == 0.
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// true in exactly one (converged) lane of the warp; code under this predicate is issued once per warp by construction, so
// the compiler needs no per-lane loop around uniform-datapath instructions such as UBLKCP
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}
// same with an L2 eviction-priority hint (createpolicy result)
__device__ __forceinline__ void bulk_g2s_hint(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar,
                                              uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}

__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// {a0, a1} += p * {v0, v1}: two IEEE fp32 fmas
__device__ __forceinline__ void ffma2(float &a0, float &a1, float p, float v0, float v1) {
    a0 = fmaf(p, v0, a0);
    a1 = fmaf(p, v1, a1);
}
// warp-wide max by butterfly shuffles (sm_90 has no f32 redux.sync); -inf lanes are neutral, no NaN inputs expected
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Programmatic dependent launch: wait for the producer grid's memory to be visible / let the
// dependent grid start its prologue.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- launch parameter blocks shared between translation units ---------------------------------
struct AppendParams {
    const __nv_bfloat16 *k_new;   // (B, Hkv, D) or null
    const __nv_bfloat16 *v_new;   // (B, Hkv, D)
    const __nv_bfloat16 *avg_k;   // (B, Hkv, D) or null (dense: no centring)
    uint8_t *rows;                // [BG][cap] records
    const int32_t *len;           // [B] length AFTER plan(): the new row goes to len-1
    int BG, Hkv, cap;
};

struct AttendParams {
    const uint8_t *kv;        // [C*Hkv][M] records        (sparse store; may be null if no sampled rows)
    const float *kn;          // [C*Hkv][M]
    const int32_t *slot_of;   // [B] slot of each request, or null: request b reads slot b
    const uint8_t *win;       // [BG][Wcap] records         (null -> no window rows)
    const int32_t *win_len;   // [B]
    const int32_t *ind;       // [H][M]
    const int32_t *nnz;       // [H]
    const __nv_bfloat16 *q;   // [H][D]
    const float *qnorm;       // [H]
    __nv_bfloat16 *out;       // [H][D]
    float *out_f32;           // [H][D] or null: the same output before the bf16 rounding (option "out_f32")
    float *mve;               // [2][H] or null: row0 = m*log2e, row1 = LSE2
    float *partials;          // [nwarps][2][PART_FLOATS]
    int32_t *counters;        // [H]
    int H, G, Hq, M, Wcap, K, L;
    unsigned long long *dbg;  // optional per-warp stage timestamps (16 x u64 per warp), null in production
    int skip;                 // measurement aid (option "attend_skip"): 1 = no row fetch, 2 = no tile math, 4 = no merges
};

// The new rows of layer ls: its window (keys centred on avg_k) or, dense, its full KV cache (in shared dense mode its request
// tails, addressed from ctx->dense_base_map() -- see launch_append_tokens).
inline AppendParams append_params(const mpig_ctx *ctx, const LayerStore &ls, const void *k, const void *v, bool dense) {
    AppendParams a = {};
    a.k_new = (const __nv_bfloat16 *)k;
    a.v_new = (const __nv_bfloat16 *)v;
    a.avg_k = dense ? nullptr : ls.avg_k;
    const bool tail = dense && ctx->dense_tail_rows > 0;
    a.rows = dense ? (tail ? ls.dense_tail : ls.dense_kv) : ls.win;
    a.len = dense ? ctx->dense_len : ctx->win_len;
    a.BG = ctx->BG;
    a.Hkv = ctx->cfg.num_key_value_heads;
    a.cap = dense ? (tail ? ctx->dense_tail_rows : ctx->cfg.max_length) : ctx->Wcap;
    return a;
}

// The fields of an attend_mma launch that every caller takes from the context.  The caller sets the rows to read (kv, kn,
// slot_of, win, win_len, ind, nnz), mve, and Wcap / K / L where they differ.
inline AttendParams attend_params(const mpig_ctx *ctx, const void *q, const float *qnorm, void *out) {
    AttendParams p = {};
    p.q = (const __nv_bfloat16 *)q;
    p.qnorm = qnorm;
    p.out = (__nv_bfloat16 *)out;
    p.out_f32 = ctx->want_out_f32 ? ctx->out_f32 : nullptr;
    p.partials = ctx->partials;
    p.counters = ctx->counters;
    p.H = ctx->H;
    p.G = ctx->G;
    p.Hq = ctx->cfg.num_attention_heads;
    p.M = ctx->cfg.max_length;
    p.Wcap = ctx->Wcap;
    p.K = ctx->cfg.K;
    p.L = ctx->cfg.L;
    return p;
}

// rows = query rows to hash (0 = B*Hq)
int launch_simhash(mpig_ctx *ctx, const void *query_bf16, int32_t *codes, float *qnorm, const AppendParams *ap,
                   cudaStream_t s, bool pdl, int rows = 0);
// the T new rows of every (request, kv-head): k/v (B, T, Hkv, d) -> rows len[b] - T + t (centred when ap.avg_k != null); with a
// base map (shared dense mode) row len[b] - T + t - base[b] of the request's tail
int launch_append_tokens(mpig_ctx *ctx, const AppendParams &ap, int T, cudaStream_t s, const int32_t *base = nullptr);
// T-token sparse decode (fused.cu): append of the T window rows, then the T-token fused kernel; q (B, T, Hq, d), k / v
// (B, T, Hkv, d), out (B, T, Hq*d).  Refuses (nothing launched) when the fused decode does not apply.
int launch_fused_tokens(mpig_ctx *ctx, int layer, int T, const void *q, const void *k, const void *v, void *out, cudaStream_t s);
// dense decode (attend_dense.cu) of the dense layer ls, T*G <= 32: T = 1 (single-token decode, causal) or the pending step's T
// (ancestor masks); q / out (B, T, Hq, d), rows already appended.  Shared dense mode (dense_tail_rows > 0) reads the slot stores
// and the request tails.
int launch_attend_dense(mpig_ctx *ctx, const LayerStore &ls, int T, const void *q, void *out, cudaStream_t s, bool pdl);
// chunk step of T tokens on layer `layer` (attend_chunk.cu): append of the T rows, then exact causal attention over the request's
// store + window (sparse) or dense rows (dense); q / out (B, T, Hq, d), k / v (B, T, Hkv, d)
int launch_chunk_attend(mpig_ctx *ctx, int layer, int T, const void *q, const void *k, const void *v, void *out, cudaStream_t s);
int chunk_partial_tiles(const mpig_ctx *ctx);
size_t chunk_partial_bytes(const mpig_ctx *ctx);
int chunk_counter_count(const mpig_ctx *ctx, int t_max);
// store_n[layer] from the host mirror n_off[layer] (an asynchronous copy of pageable memory: the values are read at the call)
int upload_store_n(mpig_ctx *ctx, int layer, cudaStream_t s);
int launch_probe(mpig_ctx *ctx, int layer, const int32_t *query, int32_t *results, int32_t *nnz, cudaStream_t s, bool pdl);
int launch_attend_mma(mpig_ctx *ctx, const AttendParams &p, cudaStream_t s, bool pdl);
int launch_fused(mpig_ctx *ctx, int layer, const void *q, const void *k, const void *v, void *out, cudaStream_t s, bool pdl,
                 const mpig_peer *peer = nullptr, int peer_rank = 0, int peer_world = 1, volatile uint32_t *host_flags = nullptr,
                 uint32_t host_epoch = 0);
bool fused_applicable(const mpig_ctx *ctx);
// clusters of C fused-kernel CTAs of `threads` threads (at the full shared-memory carve-up) the current device keeps resident
int fused_resident_clusters(int C, int threads);
int fused_cluster_waves(const mpig_ctx *ctx);   // waves of clusters one fused launch takes (0 = not applicable / unknown)
int launch_pack_nhd(mpig_ctx *ctx, const void *k, const void *v, uint8_t *rec, int Hkv, int n, int rows_cap, cudaStream_t s);
// window spill, table side (tables.cu): merge the codes of the keys [n_old[c], n_old[c] + g[c]) of every context slot c into
// its tables of `layer`.  codes (Hkv, L, g[c]) int16 per slot, slot c's block starting at pre[c] * Hkv * L; g / pre / n_old
// are device arrays [C].
int launch_table_merge(mpig_ctx *ctx, int layer, const int16_t *codes, const int32_t *g, const int32_t *pre, const int32_t *n_old,
                       cudaStream_t s);
// a compaction (store.cu): drop the keys >= lo[c] from slot c's tables of `layer`, whose keys were [0, hi[c]) (tables.cu);
// lo / hi are device arrays [C], and lo[c] == hi[c] leaves slot c untouched
int launch_table_truncate(mpig_ctx *ctx, int layer, const int32_t *lo, const int32_t *hi, cudaStream_t s);
// shared spill mode: a request's place in the visibility map changes (store.cu).  src >= 0: dst sees exactly the private keys src
// sees (a fork); src < 0: dst sees no private key (a bind).  Every slot's map is rewritten.
int launch_vis_rebind(mpig_ctx *ctx, int src, int dst, cudaStream_t s);
// shared spill mode: a fill of `layer` through request `request` (n prompt keys) empties the private region of its slot
int reset_private(mpig_ctx *ctx, int layer, int request, int n, cudaStream_t s);

// ---- host helpers --------------------------------------------------------------------------
int check_layer(mpig_ctx *ctx, int layer, bool need_sparse, const char *who);
// the device lengths of requests [b0, b0 + n) into wl (win_len) and dl (dense_len), either may be null; synchronises s.  The
// device lengths are the truth: replays of a captured plan advance only them (step.cu).
int read_lengths(const mpig_ctx *ctx, int b0, int n, int32_t *wl, int32_t *dl, cudaStream_t s);
// h_slot_of / h_dense_base from the device maps when a captured reorder may have changed them (!h_map_exact; synchronises s),
// a no-op otherwise.  Every host path that reads either mirror calls it first (context.cu).
int refresh_maps(mpig_ctx *ctx, cudaStream_t s);
inline cudaStream_t as_stream(void *s) { return (cudaStream_t)s; }

}  // namespace mpig
