// fused.cu -- ONE launch per sparse layer: SimHash -> probe -> importance-weighted gather attention (+ window, LSE merge).
//
// Replaces, for one decode token of one sparse layer, the whole of LSHSparseAttnServer.decode (models/attnserver.py:261-312):
//   :264-270  norm_q, bf16 GEMM with hash_func, sign, pack              -> phase HASH   (mma.sync m16n8k16, sign bits only)
//   :272-273  D2H of the codes, lsh.cc:210-288 batch_retrieve/retrieve    -> phase PROBE  (tag sweeps in shared memory)
//   :299-300  sparse_attention.cc:629-745 attention_wrapper              -> phase ATTEND (TMA row gather + tensor-core scores)
//   :275-296  centre + append the new K/V row, FlashInfer window decode   -> window rows join the same online softmax
//   :305-308  merge_state                                                -> the online softmax IS the LSE merge
//
// Why one kernel.  As three PDL-chained launches the layer cost 34 us at C2 (Llama-3.1-8B, n = 97 932, K10 L150) against a
// 4.3 us HBM floor: each launch paid ~2 us of launch + prologue, the probe wrote the index list and nnz to HBM and the
// attention kernel re-read them behind a partition computation and two dependent loads (6.5 us before the first record was
// requested).  Here the thread-block CLUSTER that probes q-head h also attends it:
//
//   grid = H clusters of C = S*r CTAs (S key segments -- as many as the cluster has CTAs wherever the context allows, at most
//   65 536 keys each --, r CTAs per segment); CTA c owns Mc keys of one segment.  Large batches: C = 1, several waves.
//   HASH    the cluster splits the L tables: CTA c projects norm_q on the K*ceil(L/C) columns of its tables (hash_func_t rows
//           as the A operand straight from L2 with 16-byte loads, norm_q as the one used column of B; both operands share a
//           k-permutation so no shuffles are needed), keeps the sign bits, packs K-bit codes and stores them into EVERY
//           CTA's code array through distributed shared memory; one cluster barrier.
//   PROBE   exactly the tag scheme of probe_kernel (tables.cu): bucket bounds -> 32-candidate chunks -> sweep 1 (tag = table
//           id) -> sweep 2 (SEL where another table won) -> tag in {EMPTY, id, SEL} == the reference's mask byte {0,1,2}.
//   SELECT  the SEL keys of the CTA's range are compacted (ascending) into a shared-memory list; nothing goes to HBM.
//   ATTEND  consumer warps take 16-row tiles of that list: ONE elected lane issues the 16 512-byte cp.async.bulk (TMA engine)
//           of a tile in a warp-uniform sequence, 8 warps at a time in warp order (issue window), completion counted in bytes
//           on the warp's mbarrier; scores on the tensor cores (ldmatrix + mma.m16n8k16, q in column 0), the LSH re-weighting
//           lane-per-row, online softmax in base 2 (shuffle max), PV as fp32 FMAs.  Window tiles (round-robin over the cluster)
//           take the same path; the token being decoded is built in place from k_new - avg_k / v_new: no CTA waits for an append.
//   MERGE   warp states -> CTA state (four warps, a dimension per lane) -> rank 0 (DSMEM, one cluster barrier) -> output.
// The index list and nnz are written to HBM only for mpig_last_probe (nnz always: one int per head; the list on request).
#include <algorithm>

#include "attend_common.cuh"
#include "probe_common.cuh"

namespace mpig {

constexpr int FT = 16;                 // rows per attention tile (one m16 tile)
constexpr int F_MAXCH = 1024;          // 32-candidate chunks a CTA can stream (8-byte records); longer streams -> three-launch path
// chunks per warp kept in registers between the sweeps: 256 chunks per CTA either way (a CTA owns one key segment and streams
// ~200 chunks at C2); more go through the slower overflow loops
template <int THREADS> struct FKeep { static constexpr int value = (THREADS == 1024) ? 8 : 16; };
constexpr int VSLOT = D * 2;           // KREG variant: only the V half of a record is staged in shared memory (256 B per row)

// Shared-memory carve-up (computed on the host, carried in the parameter block).
//   [ scratch: tag | chunk | tstart | tlen | tcpre | wsum | codes | bits ]   alive until the selected keys are listed
//   [ persistent: counts | q | nq | misc | sel | cpart | bars ]
//   [ slots: ncw_base row buffers ]
// Once the list exists the scratch is dead, so `n_extra` MORE row buffers are carved out of it (same stride) and handed to the
// warps ncw_base .. ncw_base + n_extra - 1: at C2 that is 26 buffers = 416 rows in flight for ~406 rows per CTA, i.e. ONE round of
// tiles instead of two.  (Not when the index list / masks are saved for mpig_last_probe, and not when the selection needs
// several passes: both read the tags again.)  A warp's partial state is stored at the start of its own buffer when it is done.
struct FusedSmem {
    uint32_t tag, chunk, tstart, tlen, tcpre, wsum, codes, bits, scratch_end, counts, q, nq, misc, sel, cpart, bars, slots, total;
    uint32_t ncw_base, n_extra;
};
inline FusedSmem fused_smem(int Mc, int tag_bytes, int L, int K, int C, int ncw_base, int max_warps, int selcap, int slot_stride) {
    FusedSmem s;
    size_t o = 0;
    auto take = [&](size_t bytes, size_t align) {
        o = (o + align - 1) & ~(align - 1);
        const size_t at = o;
        o += bytes;
        return (uint32_t)at;
    };
    s.tag = take((size_t)Mc * tag_bytes + 32, 128);   // + a dummy slot (index Mc) that absorbs the sweeps' non-candidates
    s.chunk = take((size_t)F_MAXCH * 8, 8);
    s.tstart = take((size_t)L * 4, 4);
    s.tlen = take((size_t)L * 4, 4);
    s.tcpre = take((size_t)(L + 1) * 4, 4);
    s.wsum = take(40 * 4, 4);
    s.codes = take((size_t)L * 4, 4);
    s.bits = take((size_t)((L + C - 1) / C) * K + 32, 4);
    s.scratch_end = (uint32_t)o;
    s.counts = take(16 * 4, 4);
    s.q = take(256, 16);
    s.nq = take(256, 16);
    s.misc = take(32, 16);
    s.sel = take((size_t)selcap * 2, 16);
    s.cpart = take((size_t)C * PART_FLOATS * 4, 16);
    s.bars = take((size_t)max_warps * 16, 8);   // [max_warps] rows-landed barriers | [max_warps] requests-issued barriers
    s.slots = take((size_t)ncw_base * FT * slot_stride, 128);
    s.total = (uint32_t)o;
    s.ncw_base = (uint32_t)ncw_base;
    const int fit = (int)(s.scratch_end / (uint32_t)(FT * slot_stride));
    s.n_extra = (uint32_t)std::max(0, std::min(fit, max_warps - ncw_base));
    return s;
}

struct FusedParams {
    const __nv_bfloat16 *q;        // [H][D]
    const __nv_bfloat16 *k_new;    // [BG][D]
    const __nv_bfloat16 *v_new;    // [BG][D]
    const __nv_bfloat16 *avg_k;    // [BG][D]
    const __nv_bfloat16 *hf_t;     // [K*L][D]  (hash_func transposed)
    const int32_t *codes_in;       // [H][L] or null: hash inside the kernel
    const int32_t *offsets;        // [BG][L][S][NB+1]
    const uint16_t *items;         // [BG][L][M]
    const uint8_t *kv;             // [BG][M] records
    const float *kn;               // [BG][M]
    uint8_t *win;                  // [BG][Wcap] records; row win_len-1 is WRITTEN by this kernel
    const int32_t *win_len;        // [B] (already advanced by plan())
    __nv_bfloat16 *out;            // [H][D]
    float *out_f32;                // [H][D] or null
    float *mve;                    // [2][H] or null
    int32_t *nnz_out;              // [H]
    int32_t *results_out;          // [H][M] or null
    uint32_t *bitmaps_out;         // [H][2][words] or null
    int32_t *codes_out;            // [H][L] or null
    unsigned long long *dbg;       // [grid][16] or null
    int dbg_cap;                   // CTA records the debug buffer holds
    int issue_win;                 // warps of a CTA that issue their first tile's row requests at the same time (0 = all)
    // KV-head tensor parallelism (peer.cu): when peer_blocks != null the epilogue ALSO stores each head's output row into every
    // rank's exchange block (slot [parity][peer_rank], 32 flag-carrying 16-byte lines per head) over NVLink
    // host-buffer entry point (mpig_decode_host): flags in mapped pinned memory, flag[h] = host_epoch once head h's row is out
    volatile uint32_t *host_flags;
    uint32_t host_epoch;
    uint8_t *const *peer_blocks;   // [peer_world] mapped exchange blocks, or null
    const unsigned long long *peer_local;   // [16] = epoch of this rank's exchange object (peer.cu)
    size_t peer_slot_bytes, peer_data_bytes;
    int peer_rank, peer_world;
    int H, G, Hq, M, Wcap, K, L, NB, S, r, Mc, words, ncw, selcap, C, seg_len;
    FusedSmem lay;                 // shared-memory carve-up, computed once on the host
    int ntok;                      // TOK instantiation: query tokens T per request (H = B*T*Hq virtual heads)
};

__device__ __forceinline__ unsigned long long clk64() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(t));
    return t;
}

// Block-wide exclusive scan with ONE barrier, for this kernel's issue-bound phases: warp scans -> per-warp totals in shared memory ->
// the prefix of the warp totals and the grand total by REDUX.SUM (two instructions instead of a second 5-step shuffle scan).
// Only the first `nwa` warps hold non-zero values (warp-uniform): the others skip their warp scan.  `wtot`: >= 32 ints, not reused
// before the caller's next barrier.
__device__ __forceinline__ int block_exclusive_scan_redux(int v, int *wtot, int *total, int warp, int lane, int nwa) {
    int inc = v;
    if (warp < nwa) {
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) wtot[warp] = inc;
    }
    __syncthreads();
    const int w = (lane < nwa) ? wtot[lane] : 0;
    *total = __reduce_add_sync(0xffffffffu, w);
    return __reduce_add_sync(0xffffffffu, (lane < warp) ? w : 0) + inc - v;
}

// THREADS = 1024: one CTA per SM (B*Hq*C <= #SMs);  THREADS = 512: two CTAs per SM (large batches: B*Hq*C <= 2 * #SMs), each with
// half the shared memory -- fewer row slots per CTA, the same number per SM.  64 registers per thread either way.
// KREG = true (default): the K half of every row goes from HBM straight into the mma A-fragment registers (16-byte loads with a
// k-permutation shared with the q operand, like the hash phase) and only the V half is staged in shared memory by the TMA
// engine: 256 B instead of 528 B of shared memory per row in flight, so ALL of a CTA's rows (~400 at C2) are in flight at once
// instead of ~300 in two rounds.  KREG = false: whole 512-byte records through TMA + ldmatrix (the stand-alone kernel's way).
// TOK = true: a verification step of T = gp.ntok tokens per request.  Cluster v serves VIRTUAL head v = (b*T + t)*Hq + h: q, out
// and every per-head output are indexed by v (the (B, T, Hq, d) layout), the tables / records / window of group b*Hkv + h/G are
// read, and the window ends T-1-t rows before win_len[b].  The T new rows were appended by append_tokens_kernel, so k_new is null:
// no in-kernel row build.  Of the step's rows the token sees those whose bit is set in its ancestor mask (gp.anc[b*T + t]; a chain
// sets bits 0..t, so nothing is masked): the other rows score -inf.  `anc` is a kernel argument of its own (null for the
// single-token instantiations) so that FusedParams, and with it their code, stays as it is.
// slot_of (B), or null: the tables, records and key norms are those of slot group slot_of[b]*Hkv + h/G (context slots shared by
// several requests); the window, k_new and avg_k stay those of group b*Hkv + h/G.  Null reads group b*Hkv + h/G for both.
// SPILL (shared spill mode): vis / plo are the slots' visibility maps [C][M] and this layer's private starts [C]; the private keys
// of the slot that request b does not see leave the tags before SELECT (filter_private).  Kernel arguments of their own, like anc
// and slot_of, so that FusedParams stays as it is, and null in the instantiations without SPILL, which never read them: at the
// 64-register cap any reference to them, even a test for null, moved the allocator's choices and added spills to the default
// instantiation (DESIGN.md section 3.12).
template <typename TagT, int THREADS, bool DBG, bool KREG, bool TOK = false, bool SPILL = false>
__global__ void __launch_bounds__(THREADS, (THREADS == 1024) ? 1 : 2) fused_decode_kernel(const __grid_constant__ FusedParams gp,
                                                                                                   const int32_t *__restrict__ anc,
                                                                                                   const int32_t *__restrict__ slot_of,
                                                                                                   const uint32_t *__restrict__ vis,
                                                                                                   const int32_t *__restrict__ plo) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    __shared__ FusedParams p_s;   // parameters staged once (constant-bank misses were microseconds on the critical path)
    {
        constexpr int NW32 = (int)(sizeof(FusedParams) / 4);
        for (int i = threadIdx.x; i < NW32; i += THREADS)
            reinterpret_cast<uint32_t *>(&p_s)[i] = reinterpret_cast<const uint32_t *>(&gp)[i];
    }
    // the CTA's coordinates cost five integer divisions: one thread does them (32 warps x ~170 instructions otherwise)
    __shared__ int s_geo[8];
    if (threadIdx.x == THREADS - 1) {
        const unsigned C_ = cluster_nctarank(), c_ = cluster_ctarank();
        const int h_ = blockIdx.x / C_;
        s_geo[0] = h_;
        if (TOK) {
            const int hq = h_ % gp.Hq, bt = h_ / gp.Hq, b = bt / gp.ntok;
            s_geo[1] = b * (gp.Hq / gp.G) + hq / gp.G;
            s_geo[2] = b;
            s_geo[5] = gp.ntok - 1 - (bt - b * gp.ntok);   // rows of later tokens at the end of the window
        } else {
            s_geo[1] = h_ / gp.G;
            s_geo[2] = h_ / gp.Hq;
        }
        s_geo[3] = (int)c_ / gp.r;
        s_geo[4] = ((int)c_ % gp.r) * gp.Mc;
        // slot group.  Read before griddepcontrol.wait: only copy-engine calls write the map (never a kernel), and a kernel starts
        // after every copy ordered before it in the stream has completed (PDL overlaps a kernel with a preceding kernel only)
        s_geo[6] = slot_of ? __ldg(slot_of + s_geo[2]) * (gp.Hq / gp.G) + (h_ % gp.Hq) / gp.G : s_geo[1];
        if (SPILL) s_geo[7] = __ldg(slot_of + s_geo[2]);   // shared spill mode (C < B: the map exists): the slot itself
    }
    unsigned long long t_dbg[12];
    if (DBG) {
#pragma unroll
        for (int i = 0; i < 12; ++i) t_dbg[i] = 0;
        t_dbg[0] = clk64();
    }
    __syncthreads();
    const FusedParams &p = p_s;
    constexpr TagT SEL = (TagT)(~(TagT)0);
    constexpr TagT EMPTY = (TagT)(SEL - 1);
    constexpr int NWARPS = THREADS / 32;
    const unsigned C = cluster_nctarank(), c = cluster_ctarank();
    const int h = s_geo[0], g = s_geo[1], bq = s_geo[2];   // g: the group of the window and the new row
    // the slot group of the tables, records and key norms, re-read from shared memory where it is used (volatile: a value kept
    // live across the kernel would add spills at the 64-register cap)
    auto slot_group = [&]() -> size_t { return (size_t)*reinterpret_cast<volatile int *>(&s_geo[6]); };
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // the same value, but provably warp-uniform (uniform datapath: tile loop, request issue)
    constexpr int F_KEEP = FKeep<THREADS>::value;
    const int L = p.L, K = p.K, Mc = p.Mc, M = p.M, S = p.S, r = p.r, NB = p.NB, ncw = p.ncw;
    constexpr int SSTRIDE = KREG ? VSLOT : SLOT;   // bytes per row slot
    const FusedSmem &lay = p.lay;
    TagT *tag = reinterpret_cast<TagT *>(smem_raw + lay.tag);
    int2 *s_chunk = reinterpret_cast<int2 *>(smem_raw + lay.chunk);   // per 32-candidate chunk: {item offset, table*64 + count}
    int *s_tstart = reinterpret_cast<int *>(smem_raw + lay.tstart);   // per table: bucket start / length / chunks before it (only the
    int *s_tlen = reinterpret_cast<int *>(smem_raw + lay.tlen);       // chunks past the record array look these up)
    int *s_tcpre = reinterpret_cast<int *>(smem_raw + lay.tcpre);
    int *s_counts = reinterpret_cast<int *>(smem_raw + lay.counts);
    int *wsum = reinterpret_cast<int *>(smem_raw + lay.wsum);
    int *s_codes = reinterpret_cast<int *>(smem_raw + lay.codes);
    uint8_t *s_bits = smem_raw + lay.bits;
    uint32_t *s_q32 = reinterpret_cast<uint32_t *>(smem_raw + lay.q);     // raw query row (bf16 pairs)
    uint32_t *s_nq32 = reinterpret_cast<uint32_t *>(smem_raw + lay.nq);   // normalised query row (bf16 pairs)
    float *s_misc = reinterpret_cast<float *>(smem_raw + lay.misc);       // [0] = |q| (fp32), [1] = window length (int bits)
    uint16_t *s_sel = reinterpret_cast<uint16_t *>(smem_raw + lay.sel);
    float *s_cpart = reinterpret_cast<float *>(smem_raw + lay.cpart);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + lay.bars);
    uint8_t *slots_all = smem_raw + lay.slots;

    // CTA c of the cluster owns keys [lo_key, lo_key + Mc): sub-range (c % r) of key segment (c / r)
    const int seg = s_geo[3];
    const int lo_rel = s_geo[4];
    const int lo_key = seg * p.seg_len + lo_rel;
    const bool seg_ok = seg < S;

    // ---- P0: everything that does not depend on the caller's previous kernel ------------------------------------------
    cluster_arrive_relaxed();   // paired with the wait after P1: no remote shared-memory store before every CTA has started
    {
        const uint32_t fillw = (sizeof(TagT) == 1) ? 0xFEFEFEFEu : 0xFFFEFFFEu;
        uint4 *tw = reinterpret_cast<uint4 *>(tag);   // Mc is a multiple of 32, the array 128-byte aligned
        for (int w = tid; w < (int)(Mc * sizeof(TagT) / 16); w += THREADS) tw[w] = make_uint4(fillw, fillw, fillw, fillw);
    }
    if (warp < ncw + (int)lay.n_extra && lane == 0) {
        mbar_init(&bars[warp], 1);
        mbar_init(&bars[NWARPS + warp], 1);   // "this warp's first tile has been requested" (issue window, P5)
        fence_proxy_async();
    }
    // this warp's first tile of hash_func rows: constant data, requested now so that the L2 latency overlaps the predecessor
    // kernel's tail (under PDL) and the arrival of the query row
    const int grp = lane >> 2, tig = lane & 3;
    const int hLc = (L + (int)C - 1) / (int)C;
    const int ht0 = (int)c * hLc, hntab = max(0, min(hLc, L - ht0)), hncols = hntab * K, hcol0 = ht0 * K;
    const int hntiles = (p.codes_in == nullptr) ? ((hncols + 15) >> 4) : 0;
    const int hlast_row = K * L - 1;
    uint4 ra[4], rb[4];
    if (warp < hntiles) {
        const int ra_i = min(hcol0 + warp * 16 + grp, hlast_row), rb_i = min(hcol0 + warp * 16 + grp + 8, hlast_row);
        const uint4 *pa = reinterpret_cast<const uint4 *>(p.hf_t + (size_t)ra_i * D);
        const uint4 *pb = reinterpret_cast<const uint4 *>(p.hf_t + (size_t)rb_i * D);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            ra[kk] = __ldg(pa + kk * 4 + tig);
            rb[kk] = __ldg(pb + kk * 4 + tig);
        }
    }
    pdl_launch_dependents();
    pdl_wait();   // q / k_new / v_new come from the caller's previous kernel
    if (DBG) t_dbg[1] = clk64();

    // ---- P1: query row, its norms, the window length; the group's first head appends the new row for LATER steps --------
    if (warp == 0) {
        const uint2 v = __ldg(reinterpret_cast<const uint2 *>(p.q + (size_t)h * D) + lane);
        const float x0 = bf16lo(v.x), x1 = bf16hi(v.x), x2 = bf16lo(v.y), x3 = bf16hi(v.y);
        const float ss = warp_sum(x0 * x0 + x1 * x1 + x2 * x2 + x3 * x3);
        const float nrm32 = sqrtf(ss);                                      // fp32 norm (attnserver.py:300)
        const float nrm = bf16_bits_to_f32(f32_to_bf16_rne(nrm32));         // bf16 arithmetic exactly as torch (:265-266)
        uint2 o;
        o.x = (uint32_t)f32_to_bf16_rne(x0 / nrm) | ((uint32_t)f32_to_bf16_rne(x1 / nrm) << 16);
        o.y = (uint32_t)f32_to_bf16_rne(x2 / nrm) | ((uint32_t)f32_to_bf16_rne(x3 / nrm) << 16);
        reinterpret_cast<uint2 *>(s_q32)[lane] = v;
        reinterpret_cast<uint2 *>(s_nq32)[lane] = o;
        if (lane == 0) s_misc[0] = nrm32;
    } else if (warp == 1) {
        const int wl = p.win ? min(max(__ldg(p.win_len + bq) - (TOK ? s_geo[5] : 0), 0), p.Wcap) : 0;
        if (lane == 0) s_misc[1] = __int_as_float(wl);
        if (TOK && lane == 0) {   // first window row of the step as this token sees it, and the token's ancestor mask
            const int tk = p.ntok - 1 - s_geo[5], bt = bq * p.ntok + tk;
            s_misc[2] = __int_as_float(wl - 1 - tk);
            s_misc[3] = __int_as_float(__ldg(anc + bt));
        }
        if (c == 0 && (h % p.G) == 0 && wl > 0 && p.k_new) {
            // centred key (bf16 arithmetic as torch: fp32 subtract, RNE) | value -> window row wl-1 (attnserver.py:275-290)
            const uint2 kk = __ldg(reinterpret_cast<const uint2 *>(p.k_new + (size_t)g * D) + lane);
            const uint2 av = __ldg(reinterpret_cast<const uint2 *>(p.avg_k + (size_t)g * D) + lane);
            const uint2 vv = __ldg(reinterpret_cast<const uint2 *>(p.v_new + (size_t)g * D) + lane);
            uint2 ko;
            ko.x = (uint32_t)f32_to_bf16_rne(bf16lo(kk.x) - bf16lo(av.x)) | ((uint32_t)f32_to_bf16_rne(bf16hi(kk.x) - bf16hi(av.x)) << 16);
            ko.y = (uint32_t)f32_to_bf16_rne(bf16lo(kk.y) - bf16lo(av.y)) | ((uint32_t)f32_to_bf16_rne(bf16hi(kk.y) - bf16hi(av.y)) << 16);
            uint8_t *rec = p.win + ((size_t)g * p.Wcap + (wl - 1)) * REC;
            *reinterpret_cast<uint2 *>(rec + 8 * lane) = ko;
            *reinterpret_cast<uint2 *>(rec + 2 * D + 8 * lane) = vv;
        }
    }
    __syncthreads();
    cluster_wait();   // (arrived at kernel entry) every CTA of the cluster is running: distributed shared memory may be written
    const int wlen = __float_as_int(s_misc[1]);
    // ---- P2: HASH (this CTA's share of the tables), codes exchanged through distributed shared memory ------------------
    if (p.codes_in == nullptr) {
        const int t0 = ht0, ntab = hntab;
        for (int nt = warp; nt < hntiles; nt += NWARPS) {
            // A = 16 columns of hash_func (rows of hash_func_t); lane (grp, tig) fetches 16 B = 8 consecutive k of rows grp and
            // grp+8 per 32-k block: physical k (kk*32 + tig*8 + 0..7) feeds the two mma of that block, the same permutation
            // on the B side (norm_q) -- the contraction does not care about the order of k.
            if (nt != warp) {   // the first tile was requested in P0
                const int ra_i = min(hcol0 + nt * 16 + grp, hlast_row), rb_i = min(hcol0 + nt * 16 + grp + 8, hlast_row);
                const uint4 *pa = reinterpret_cast<const uint4 *>(p.hf_t + (size_t)ra_i * D);
                const uint4 *pb = reinterpret_cast<const uint4 *>(p.hf_t + (size_t)rb_i * D);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    ra[kk] = __ldg(pa + kk * 4 + tig);
                    rb[kk] = __ldg(pb + kk * 4 + tig);
                }
            }
            float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                uint4 qv = make_uint4(0u, 0u, 0u, 0u);
                if (grp == 0) qv = reinterpret_cast<const uint4 *>(s_nq32)[kk * 4 + tig];   // column 0 of B
                const uint32_t a1[4] = {ra[kk].x, rb[kk].x, ra[kk].y, rb[kk].y};
                const uint32_t a2[4] = {ra[kk].z, rb[kk].z, ra[kk].w, rb[kk].w};
                mma_16816(c0, c1, c2, c3, a1, qv.x, qv.y);
                mma_16816(c0, c1, c2, c3, a2, qv.z, qv.w);
            }
            if (tig == 0) {   // column 0: only the SIGN survives (attnserver.py:267 .gt(0))
                s_bits[nt * 16 + grp] = (uint8_t)(c0 > 0.f);
                s_bits[nt * 16 + grp + 8] = (uint8_t)(c2 > 0.f);
            }
        }
        __syncthreads();
        {   // little-endian pack per table (attnserver.py:268-270): a warp takes floor(32 / K) tables at a time, lane i reads
            // sign bit i of the group and ONE ballot assembles the codes (K <= 15, checked by the host)
            const int tpw = 32 / K;
            for (int tb = warp * tpw; tb < ntab; tb += NWARPS * tpw) {
                const int nt_here = min(tpw, ntab - tb);
                const unsigned m = __ballot_sync(0xffffffffu, lane < nt_here * K && s_bits[tb * K + lane] != 0);
                if (lane < nt_here) {
                    const int code = (int)((m >> (lane * K)) & ((1u << K) - 1u));
                    for (unsigned rr = 0; rr < C; ++rr) st_shared_cluster_u32(&s_codes[t0 + tb + lane], rr, (uint32_t)code);
                    if (p.codes_out) p.codes_out[(size_t)h * L + t0 + tb + lane] = code;
                }
            }
        }
        cluster_barrier();
    } else {
        for (int t = tid; t < L; t += THREADS) s_codes[t] = __ldg(p.codes_in + (size_t)h * L + t);
        __syncthreads();
    }
    if (DBG) t_dbg[2] = clk64();

    // ---- P3: PROBE (lsh.cc:243-288) -- the tag scheme of probe_kernel (tables.cu), trimmed for instruction count: this phase
    //      turned out ISSUE-bound (ncu: 42 % issue-slot utilisation over the whole kernel, the sweeps and the compaction alone
    //      were half of the 11.5 M warp instructions), so everything a candidate chunk needs is precomputed into ONE 8-byte record.
    int total_chunks = 0;
    {
        int my_chunks[(1024 + THREADS - 1) / THREADS], my_start[(1024 + THREADS - 1) / THREADS], my_len[(1024 + THREADS - 1) / THREADS];
#pragma unroll
        for (int rr = 0; rr < (1024 + THREADS - 1) / THREADS; ++rr) {
            const int t = tid + rr * THREADS;
            my_chunks[rr] = my_start[rr] = my_len[rr] = 0;
            if (t < L) {
                const int code = s_codes[t];
                int s = 0, e = 0;
                if (seg_ok && code >= 0 && code < NB) {
                    const int32_t *o = p.offsets + ((slot_group() * L + t) * S + seg) * (size_t)(NB + 1) + code;
                    s = __ldg(o);
                    e = __ldg(o + 1);
                }
                my_start[rr] = s;
                my_len[rr] = max(e - s, 0);
                my_chunks[rr] = (my_len[rr] + 31) >> 5;
            }
        }
#pragma unroll
        for (int rr = 0; rr < (1024 + THREADS - 1) / THREADS; ++rr) {
            if (rr * THREADS < L) {  // uniform across the CTA
                int tot_r;
                const int ex = block_exclusive_scan_redux(my_chunks[rr], wsum, &tot_r, warp, lane, min(NWARPS, (L - rr * THREADS + 31) >> 5));
                const int t = tid + rr * THREADS;
                if (t < L) {
                    s_tstart[t] = my_start[rr];
                    s_tlen[t] = my_len[rr];
                    s_tcpre[t] = total_chunks + ex;
                }
                // chunk records of table t: {offset of the chunk's first item in items_g, t * 64 + number of items (1..32)}
                for (int j = 0; j < my_chunks[rr]; ++j) {
                    const int ch = total_chunks + ex + j;
                    if (ch < F_MAXCH) s_chunk[ch] = make_int2(t * M + my_start[rr] + 32 * j, t * 64 + min(32, my_len[rr] - 32 * j));
                }
                total_chunks += tot_r;
                if ((1024 + THREADS - 1) / THREADS > 1) __syncthreads();   // wsum is reused by the next round
            }
        }
        if (tid == 0) s_tcpre[L] = total_chunks;
        // the records a warp keeps in registers (F_KEEP per warp) always exist: empty ones past the stream's end
        for (int ch = total_chunks + tid; ch < F_KEEP * NWARPS; ch += THREADS) s_chunk[ch] = make_int2(0, 0);
        __syncthreads();
    }
    if (DBG) t_dbg[3] = clk64();
    {
        const uint16_t *items_g = p.items + slot_group() * L * (size_t)M;
        const int nch = total_chunks;
        // record of chunk ch: from the array, or -- for pathologically long candidate streams -- rebuilt from the per-table data
        auto chunk_rec = [&](int ch) -> int2 {
            if (ch < F_MAXCH) return s_chunk[ch];
            int lo = 0, hi = L;
            while (hi - lo > 1) {
                const int mid = (lo + hi) >> 1;
                if (s_tcpre[mid] <= ch) lo = mid; else hi = mid;
            }
            const int j = ch - s_tcpre[lo];
            return make_int2(lo * M + s_tstart[lo] + 32 * j, lo * 64 + min(32, s_tlen[lo] - 32 * j));
        };
        // One-byte tags hold table ids 0..252; more tables are probed in passes of TPP tables: between passes every id still
        // standing ("hit exactly once so far") becomes ONE, and a later hit on ONE or SEL yields SEL.  L <= 253: a single pass,
        // identical to the scheme of probe_kernel.
        constexpr int TPP = 253;
        constexpr TagT ONE = (TagT)0xFD;
        const int npass = (L + TPP - 1) / TPP;
        if (npass == 1) {
            // L <= 253 (every BASELINE shape but ProLong's L = 300): the same two sweeps written for instruction count -- the phase
            // is ISSUE-bound (32 warps x ~330 instructions = 1.3 us per scheduler before this version).  A candidate is one
            // 32-bit word: key - first key of the range (unsigned: anything that is not this CTA's candidate is >= Mc).
            static_assert(F_KEEP * NWARPS <= F_MAXCH, "the register window lies inside the record array");
            const uint16_t *items_lane = items_g + lane;
            uint32_t raw[F_KEEP];
#pragma unroll
            for (int k = 0; k < F_KEEP; ++k) {
                const int2 rec = s_chunk[warp + k * NWARPS];   // (padded with empty records: no bounds test)
                raw[k] = 0xFFFFFFFFu;
                if (lane < (rec.y & 63)) raw[k] = (uint32_t)__ldg(items_lane + (uint32_t)rec.x);   // no use of the value here: all loads in flight
            }
#pragma unroll
            for (int k = 0; k < F_KEEP; ++k) {
                // branch-free: whatever is not a candidate of this CTA's key range goes to the dummy slot tag[Mc]
                raw[k] = min(raw[k] - (uint32_t)lo_rel, (uint32_t)Mc);
                tag[raw[k]] = (TagT)(s_chunk[warp + k * NWARPS].y >> 6);   // 0 -> 1 (lsh.cc:276-277)
            }
            for (int ch = warp + ((warp + F_KEEP * NWARPS <= F_MAXCH) ? F_KEEP * NWARPS : 0); ch < nch; ch += NWARPS) {
                if (ch < F_MAXCH && ch < warp + F_KEEP * NWARPS) continue;   // handled from registers
                const int2 rec = chunk_rec(ch);
                if (lane < (rec.y & 63)) {
                    const uint32_t i = (uint32_t)__ldg(items_g + rec.x + lane) - (uint32_t)lo_rel;
                    if (i < (uint32_t)Mc) tag[i] = (TagT)(rec.y >> 6);
                }
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < F_KEEP; ++k)
                if (tag[raw[k]] != (TagT)(s_chunk[warp + k * NWARPS].y >> 6)) tag[raw[k]] = SEL;   // 1 -> 2 (the dummy slot: anything)
            for (int ch = warp + ((warp + F_KEEP * NWARPS <= F_MAXCH) ? F_KEEP * NWARPS : 0); ch < nch; ch += NWARPS) {
                if (ch < F_MAXCH && ch < warp + F_KEEP * NWARPS) continue;
                const int2 rec = chunk_rec(ch);
                if (lane < (rec.y & 63)) {
                    const uint32_t i = (uint32_t)__ldg(items_g + rec.x + lane) - (uint32_t)lo_rel;
                    if (i < (uint32_t)Mc && tag[i] != (TagT)(rec.y >> 6)) tag[i] = SEL;
                }
            }
            __syncthreads();
        } else
        for (int ps = 0; ps < npass; ++ps) {
            const int T0 = ps * TPP;
            const int ch0 = (npass == 1) ? 0 : s_tcpre[T0], ch1 = (npass == 1) ? nch : s_tcpre[min(L, T0 + TPP)];
            int idx[F_KEEP];
            // every load of the bucket stream is issued before the first tag is written: the stream costs one memory latency
#pragma unroll
            for (int k = 0; k < F_KEEP; ++k) {
                const int ch = ch0 + warp + k * NWARPS;
                idx[k] = -1;
                if (ch < ch1 && ch < F_MAXCH) {
                    const int2 rec = s_chunk[ch];
                    if (lane < (rec.y & 63)) idx[k] = (int)__ldg(items_g + rec.x + lane);   // NO use of the value here: all loads in flight
                }
            }
#pragma unroll
            for (int k = 0; k < F_KEEP; ++k) {
                const int ch = ch0 + warp + k * NWARPS;
                const int i = idx[k] - lo_rel;   // key - first key of this CTA's range
                idx[k] = (idx[k] >= 0 && i >= 0 && i < Mc) ? i : -1;   // keep only this CTA's key range
                if (idx[k] >= 0) {
                    const TagT id = (TagT)((s_chunk[ch].y >> 6) - T0);
                    if (ps == 0) {
                        tag[idx[k]] = id;   // 0 -> 1 (lsh.cc:276-277)
                    } else {
                        const TagT v = tag[idx[k]];
                        tag[idx[k]] = (v == ONE || v == SEL) ? SEL : id;
                    }
                }
            }
            // beyond the register window / the record array (long candidate streams)
            for (int ch = ch0 + warp + ((ch0 + warp + F_KEEP * NWARPS <= F_MAXCH) ? F_KEEP * NWARPS : 0); ch < ch1; ch += NWARPS) {
                if (ch < F_MAXCH && ch < ch0 + warp + F_KEEP * NWARPS) continue;   // handled from registers
                const int2 rec = chunk_rec(ch);
                if (lane < (rec.y & 63)) {
                    const int i = (int)__ldg(items_g + rec.x + lane) - lo_rel;
                    if (i >= 0 && i < Mc) {
                        const TagT id = (TagT)((rec.y >> 6) - T0);
                        const TagT v = tag[i];
                        tag[i] = (ps > 0 && (v == ONE || v == SEL)) ? SEL : id;
                    }
                }
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < F_KEEP; ++k) {
                const int ch = ch0 + warp + k * NWARPS;
                if (idx[k] >= 0 && tag[idx[k]] != (TagT)((s_chunk[ch].y >> 6) - T0)) tag[idx[k]] = SEL;  // 1 -> 2
            }
            for (int ch = ch0 + warp + ((ch0 + warp + F_KEEP * NWARPS <= F_MAXCH) ? F_KEEP * NWARPS : 0); ch < ch1; ch += NWARPS) {
                if (ch < F_MAXCH && ch < ch0 + warp + F_KEEP * NWARPS) continue;
                const int2 rec = chunk_rec(ch);
                if (lane < (rec.y & 63)) {
                    const int i = (int)__ldg(items_g + rec.x + lane) - lo_rel;
                    if (i >= 0 && i < Mc && tag[i] != (TagT)((rec.y >> 6) - T0)) tag[i] = SEL;
                }
            }
            __syncthreads();
            if (ps + 1 < npass) {   // ids of this pass -> ONE
                uint32_t *tw = reinterpret_cast<uint32_t *>(tag);
                for (int w = tid; w < Mc / 4; w += THREADS) {
                    const uint32_t x = tw[w];
                    const uint32_t lt = __vcmpltu4(x, 0xFDFDFDFDu);   // 0xFF in every byte that holds a table id
                    tw[w] = (x & ~lt) | (0xFDFDFDFDu & lt);
                }
                __syncthreads();
            }
        }
    }
    // shared spill mode: the other requests' private keys leave the tags (after the last sweep's barrier; vis is kernel-written
    // data, and this is long after griddepcontrol.wait).  The slot comes from shared memory: nothing stays live in registers.
    if (SPILL) {
        const volatile int *vg = s_geo;
        const int sl = vg[7];
        filter_private(tag, vis + (size_t)sl * p.M, __ldg(plo + sl), vg[3] * p.seg_len + vg[4], p.Mc, vg[2]);
    }
    if (DBG) t_dbg[4] = clk64();

    // ---- P4: SELECT -- every thread owns a run of pw <= 31 tag words (odd stride: bank-conflict free) and turns it into a bit
    //      mask of its SEL keys (one bit per key, two 64-bit registers); count = popcount, ascending order = thread order.
    //      Nothing of this stays live across the attention tiles: a later pass (selection larger than the list) or the optional
    //      index-list output simply recomputes it.
    static_assert(sizeof(TagT) == 1, "the fused kernel keeps one-byte tags");
    constexpr int TPW = 4;
    const uint32_t *tagw = reinterpret_cast<const uint32_t *>(tag);
    // m7(x): bit 7 of byte b of the result is set  <=>  byte b of x is 0xFF (its low 7 bits carry into bit 7 and bit 7 is set)
    auto m7 = [](uint32_t x) -> uint32_t { return ((x & 0x7F7F7F7Fu) + 0x01010101u) & x & 0x80808080u; };
    const int sel_nwords = Mc / TPW;
    const int sel_pw = ((sel_nwords + THREADS - 1) / THREADS) | 1;
    const int sel_w0 = min(tid * sel_pw, sel_nwords), sel_w1 = min(sel_w0 + sel_pw, sel_nwords);
    auto select_count = [&]() -> int {
        int cnt = 0;
        for (int w = sel_w0; w < sel_w1; ++w) cnt += __popc(m7(tagw[w]));
        return cnt;
    };
    // calls put(ordinal, key relative to the CTA's range) for every SEL key of this thread's run, ascending
    auto select_emit = [&](int pp, auto &&put) {
        for (int w = sel_w0; w < sel_w1; ++w)
            for (uint32_t m = m7(tagw[w]); m; m &= m - 1, ++pp) put(pp, w * TPW + ((__ffs((int)m) - 1) >> 3));
    };
    if (DBG) t_dbg[5] = clk64();

    // ---- P5: ATTEND -- this CTA's window tiles (round-robin over the cluster) + its selected rows, 16-row tiles ----------
    const int nwt = (wlen + FT - 1) / FT;
    const int nwt_c = (nwt > (int)c) ? (nwt - (int)c + (int)C - 1) / (int)C : 0;
    float m_run = -CUDART_INF_F, l_run = 0.f;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    uint32_t phase = 0;
    // row buffer of this warp: one of the ncw base buffers, or one carved out of the (by then dead) probe scratch
    uint8_t *slots = (warp < ncw) ? slots_all + (size_t)warp * FT * SSTRIDE : smem_raw + (size_t)(warp - ncw) * FT * SSTRIDE;
    int ncw_eff = ncw;   // consumer warps of this CTA (decided once the selection size is known)
    uint64_t *bar = bars + warp;
    const float inv_sqrt_dim = rsqrtf((float)D);
    const float Lf = (float)L;
    const float qn = s_misc[0];
    const uint32_t a_lane_off = (uint32_t)(((lane & 7) + ((lane >> 3) & 1) * 8) * SLOT + (lane >> 4) * 16);
    const int selcap = p.selcap;

    int tot = 0;
    for (int base = 0; base == 0 || base < tot; base += selcap) {
        {   // list the selected keys with ordinal in [base, base + selcap): count, one-barrier scan, then one loop iteration per
            // SELECTED key of the thread (threads without one skip the second look at their words)
            if (sel_pw <= 8) {   // (uniform) a run of <= 32 keys: ONE look at the tags, the SEL keys as a bit mask in a register
                uint32_t nib = 0;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    // bits 7/15/23/31 of m7 -> one nibble.  Branch-free: the load may run past this thread's run (the next
                    // thread's words, or the first bytes behind the tags) -- those words are masked out below, not skipped.
                    // m7 * 0x00204081 puts the four flags at bits 28..31 (partial products on distinct bits: no carries)
                    const uint32_t pr = m7(tagw[sel_w0 + i]) * 0x00204081u;
                    nib |= (i == 7) ? (pr & 0xF0000000u) : ((pr >> (28 - 4 * i)) & (0xFu << (4 * i)));
                }
                if (sel_w1 - sel_w0 < 8) nib &= (1u << (4 * (sel_w1 - sel_w0))) - 1u;   // words past this thread's run
                const int cnt = __popc(nib);
                const int pp0 = block_exclusive_scan_redux(cnt, wsum, &tot, warp, lane, NWARPS);
                if (cnt > 0 && pp0 < base + selcap && pp0 + cnt > base) {
                    int pp = pp0;
                    for (uint32_t m = nib; m; m &= m - 1, ++pp)
                        if (pp >= base && pp < base + selcap) s_sel[pp - base] = (uint16_t)(sel_w0 * TPW + __ffs((int)m) - 1);
                }
            } else {
                const int cnt = select_count();
                const int pp0 = block_exclusive_scan_1bar(cnt, wsum, &tot);
                if (cnt > 0 && pp0 < base + selcap && pp0 + cnt > base)
                    select_emit(pp0, [&](int pp, int key) {
                        if (pp >= base && pp < base + selcap) s_sel[pp - base] = (uint16_t)key;
                    });
            }
        }
        __syncthreads();
        if (DBG && base == 0) t_dbg[6] = clk64();
        const int nsel = max(0, min(selcap, tot - base));
        const int nwin_tiles = (base == 0) ? nwt_c : 0;
        const int ntile = nwin_tiles + (nsel + FT - 1) / FT;
        if (base == 0 && tot <= selcap && p.results_out == nullptr && p.bitmaps_out == nullptr) ncw_eff = ncw + (int)lay.n_extra;
        if (warp < ncw_eff) {
            if (warp >= ncw) fence_proxy_async();   // the scratch this buffer aliases was last touched through the generic proxy
            for (int j = warp; j < ntile; j += ncw_eff) {
                const bool is_win = j < nwin_tiles;
                int row0, nrows, new_lane = -1;
                if (is_win) {
                    row0 = ((int)c + j * (int)C) * FT;
                    nrows = min(FT, wlen - row0);
                    if (row0 + nrows == wlen && p.k_new) new_lane = nrows - 1;   // the row of the token being decoded
                } else {
                    row0 = (j - nwin_tiles) * FT;
                    nrows = min(FT, nsel - row0);
                }
                float meta = -1.0f;
                float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
                if (KREG) {
                    // ---- V halves by TMA into 256-byte slots, K halves straight into the A fragments ----------------------------
                    if (lane == 0) mbar_arrive_expect_tx(bar, (uint32_t)(nrows - (new_lane >= 0 ? 1 : 0)) * VSLOT);
                    __syncwarp();
                    // record address of a row of this tile (rows past nrows alias row 0: their scores are never used)
                    auto rec_of = [&](int rr_) -> const uint8_t * {
                        const int r_ = (rr_ < nrows) ? rr_ : 0;
                        if (is_win) return p.win + ((size_t)g * p.Wcap + row0 + r_) * REC;
                        return p.kv + (slot_group() * M + (lo_key + (int)s_sel[row0 + r_])) * REC;
                    };
                    if (lane < nrows) {
                        const uint8_t *rec = rec_of(lane);
                        if (lane != new_lane) bulk_g2s(slots + (size_t)lane * VSLOT, rec + D * 2, VSLOT, bar);
                        if (!is_win) meta = __ldg(p.kn + slot_group() * M + (lo_key + (int)s_sel[row0 + lane]));
                    }
                    // lane (grp, tig): 16 B = 8 consecutive k of rows grp and grp+8 per 32-k block (4 blocks): all 8 loads in flight
                    uint4 ka[4], kb[4];
                    {
                        const uint4 *pa = reinterpret_cast<const uint4 *>(rec_of(grp));
                        const uint4 *pb = reinterpret_cast<const uint4 *>(rec_of(grp + 8));
#pragma unroll
                        for (int kk = 0; kk < 4; ++kk) {
                            ka[kk] = __ldg(pa + kk * 4 + tig);
                            kb[kk] = __ldg(pb + kk * 4 + tig);
                        }
                    }
                    if (new_lane >= 0) {   // the token being decoded: K = k_new - avg_k (bf16 arithmetic as torch), V = v_new, built in place
                        const uint2 vv = __ldg(reinterpret_cast<const uint2 *>(p.v_new + (size_t)g * D) + lane);
                        *reinterpret_cast<uint2 *>(slots + (size_t)new_lane * VSLOT + 8 * lane) = vv;
                        if (grp == new_lane || grp + 8 == new_lane) {
                            const uint4 *pk = reinterpret_cast<const uint4 *>(p.k_new + (size_t)g * D);
                            const uint4 *pv = reinterpret_cast<const uint4 *>(p.avg_k + (size_t)g * D);
#pragma unroll
                            for (int kk = 0; kk < 4; ++kk) {
                                const uint4 x = __ldg(pk + kk * 4 + tig), y = __ldg(pv + kk * 4 + tig);
                                uint4 o;
                                o.x = (uint32_t)f32_to_bf16_rne(bf16lo(x.x) - bf16lo(y.x)) | ((uint32_t)f32_to_bf16_rne(bf16hi(x.x) - bf16hi(y.x)) << 16);
                                o.y = (uint32_t)f32_to_bf16_rne(bf16lo(x.y) - bf16lo(y.y)) | ((uint32_t)f32_to_bf16_rne(bf16hi(x.y) - bf16hi(y.y)) << 16);
                                o.z = (uint32_t)f32_to_bf16_rne(bf16lo(x.z) - bf16lo(y.z)) | ((uint32_t)f32_to_bf16_rne(bf16hi(x.z) - bf16hi(y.z)) << 16);
                                o.w = (uint32_t)f32_to_bf16_rne(bf16lo(x.w) - bf16lo(y.w)) | ((uint32_t)f32_to_bf16_rne(bf16hi(x.w) - bf16hi(y.w)) << 16);
                                if (grp == new_lane) ka[kk] = o; else kb[kk] = o;
                            }
                        }
                    }
                    // scores: K_tile (16 x 128) . q on the tensor cores; q in column 0 of B with the same k-permutation; two
                    // independent accumulation chains
                    float d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        uint4 qv = make_uint4(0u, 0u, 0u, 0u);
                        if (grp == 0) qv = reinterpret_cast<const uint4 *>(s_q32)[kk * 4 + tig];
                        const uint32_t a1[4] = {ka[kk].x, kb[kk].x, ka[kk].y, kb[kk].y};
                        const uint32_t a2[4] = {ka[kk].z, kb[kk].z, ka[kk].w, kb[kk].w};
                        mma_16816(c0, c1, c2, c3, a1, qv.x, qv.y);
                        mma_16816(d0, d1, d2, d3, a2, qv.z, qv.w);
                    }
                    c0 += d0;
                    c2 += d2;
                    __syncwarp();
                    mbar_wait(bar, phase);   // V rows landed (needed from the PV loop on)
                    phase ^= 1;
                } else {
                unsigned long long w_dbg[4];
                // Issue window.  A warp issues its 16 row requests one after the other (ELECT / R2UR / UBLKCP per lane, ~77 cycles
                // each when alone = 0.65 us per tile), while the SM takes one 512-byte request every ~8 cycles from however many
                // warps offer one.  With all 26 warps issuing at once every tile completes at the END of the CTA's ~3 us issue
                // window and all tiles are computed at the same time behind it; with issue_win warps issuing at a time, in warp
                // order, the request rate is the same but tiles land -- and are computed -- one after the other while the later
                // requests are still going out (measured: 22.5 -> 20.7 us per layer at C2 with 8).  Warp w waits for warp
                // w - issue_win on that warp's "issued" mbarrier (hardware-suspended wait, no polling).
                if (p.issue_win > 0 && j == warp && base == 0 && warp >= p.issue_win) mbar_wait(bars + NWARPS + warp - p.issue_win, 0);
                if (DBG) w_dbg[0] = clk64();
                if (lane == 0) mbar_arrive_expect_tx(bar, (uint32_t)(nrows - (new_lane >= 0 ? 1 : 0)) * REC);
                __syncwarp();
                // lane r holds the record address of row r; the requests go out from ONE elected lane in an unrolled, warp-uniform
                // sequence (address broadcast by shuffle: 2 SHFL + 2 R2UR + UBLKCP per row, independent of each other) -- a
                // `cp.async.bulk` per lane compiles into a serial ELECT / R2UR.BROADCAST / UBLKCP / branch loop of ~77 cycles per row
                const uint8_t *src = nullptr;
                if (lane < nrows) {
                    if (is_win) {
                        src = p.win + ((size_t)g * p.Wcap + row0 + lane) * REC;
                    } else {
                        const int idx = lo_key + (int)s_sel[row0 + lane];
                        src = p.kv + (slot_group() * M + idx) * REC;
                        meta = __ldg(p.kn + slot_group() * M + idx);   // consumed after the scores: overlaps the row fetch
                    }
                }
                {
                    const bool leader = elect_one();
#pragma unroll
                    for (int rr = 0; rr < FT; ++rr) {
                        const uint8_t *sr = reinterpret_cast<const uint8_t *>(__shfl_sync(0xffffffffu, (unsigned long long)src, rr));
                        if (rr < nrows && rr != new_lane && leader) bulk_g2s(slots + (size_t)rr * SLOT, sr, REC, bar);
                    }
                }
                if (new_lane >= 0) {   // built in place: k_new - avg_k | v_new (every CTA that owns this tile does it itself)
                    const uint2 kk = __ldg(reinterpret_cast<const uint2 *>(p.k_new + (size_t)g * D) + lane);
                    const uint2 av = __ldg(reinterpret_cast<const uint2 *>(p.avg_k + (size_t)g * D) + lane);
                    const uint2 vv = __ldg(reinterpret_cast<const uint2 *>(p.v_new + (size_t)g * D) + lane);
                    uint2 ko;
                    ko.x = (uint32_t)f32_to_bf16_rne(bf16lo(kk.x) - bf16lo(av.x)) | ((uint32_t)f32_to_bf16_rne(bf16hi(kk.x) - bf16hi(av.x)) << 16);
                    ko.y = (uint32_t)f32_to_bf16_rne(bf16lo(kk.y) - bf16lo(av.y)) | ((uint32_t)f32_to_bf16_rne(bf16hi(kk.y) - bf16hi(av.y)) << 16);
                    *reinterpret_cast<uint2 *>(slots + (size_t)new_lane * SLOT + 8 * lane) = ko;
                    *reinterpret_cast<uint2 *>(slots + (size_t)new_lane * SLOT + 2 * D + 8 * lane) = vv;
                }
                __syncwarp();
                if (p.issue_win > 0 && j == warp && base == 0 && lane == 0) mbar_arrive_relaxed(bars + NWARPS + warp);
                if (DBG) w_dbg[1] = clk64();
                mbar_wait(bar, phase);
                phase ^= 1;
                if (DBG) {   // per-warp stamps of the first tile of CTAs 0..15: issue start / requests out / rows landed
                    w_dbg[2] = clk64();
                    if (p.dbg && lane == 0 && j == warp && blockIdx.x < 16 && base == 0) {
                        unsigned long long *wr = p.dbg + ((size_t)(gridDim.x + blockIdx.x * 32 + warp)) * 16;
                        if (gridDim.x + blockIdx.x * 32 + warp < (unsigned)p.dbg_cap) {
                            wr[0] = w_dbg[0]; wr[1] = w_dbg[1]; wr[2] = w_dbg[2]; wr[3] = (unsigned long long)nrows; wr[4] = is_win ? 1ull : 0ull;
                            wr[5] = t_dbg[6];
                        }
                    }
                }

                // scores: K_tile (16 x 128) . q on the tensor cores, q in column 0 of B
                const uint32_t slots_s = smem_u32(slots);
                float d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;   // two independent accumulation chains (4 dependent mma each)
#pragma unroll
                for (int ks = 0; ks < 8; ++ks) {
                    uint32_t a[4];
                    ldsm_x4(a, slots_s + (uint32_t)(ks * 32) + a_lane_off);
                    uint32_t b0 = 0u, b1 = 0u;
                    if (grp == 0) {
                        b0 = s_q32[ks * 8 + tig];
                        b1 = s_q32[ks * 8 + 4 + tig];
                    }
                    if (ks & 1) mma_16816(d0, d1, d2, d3, a, b0, b1);
                    else mma_16816(c0, c1, c2, c3, a, b0, b1);
                }
                c0 += d0;
                c2 += d2;
                }
                // row r < 8: c0 of lane 4r; row r >= 8: c2 of lane 4(r-8)
                const float g0 = __shfl_sync(0xffffffffu, c0, 4 * (lane & 7));
                const float g1 = __shfl_sync(0xffffffffu, c2, 4 * (lane & 7));
                const float s_mine = (lane & 8) ? g1 : g0;
                // (debug instantiation) stamps inside the first tile of the warps of CTAs 0..15: [10] scores, [11] weights, [12] softmax
                unsigned long long *wrec = nullptr;
                if (DBG && !KREG && p.dbg && lane == 0 && j == warp && blockIdx.x < 16 && base == 0 &&
                    gridDim.x + blockIdx.x * 32 + warp < (unsigned)p.dbg_cap)
                    wrec = p.dbg + ((size_t)(gridDim.x + blockIdx.x * 32 + warp)) * 16;
                if (DBG && wrec) wrec[10] = clk64() + (unsigned long long)(s_mine == 123.456f);

                // LSH-probability re-weighting (transform_kernel, sparse_attention.cc:173-183); window rows: plain s/sqrt(d)
                float z = -CUDART_INF_F;
                if (lane < nrows) {
                    z = s_mine * inv_sqrt_dim;
                    if (meta >= 0.f) {
                        float cs = s_mine / (qn * meta);
                        cs = fminf(fmaxf(cs, -1.0f), 1.0f);  // the reference would produce NaN past +-1
                        const float theta = fast_acosf(cs);
                        const float proba = 1.0f - theta * 0.318309886183790672f;
                        const float w = sample_weight(proba, K, L, Lf);
                        z -= __logf(w + 1e-4f);
                    }
                    if (TOK && is_win) {   // a step row of a node that is not this token or one of its ancestors
                        const int o = row0 + lane - __float_as_int(s_misc[2]);
                        if (o >= 0 && !((__float_as_uint(s_misc[3]) >> o) & 1u)) z = -CUDART_INF_F;
                    }
                }
                if (DBG && wrec) wrec[11] = clk64() + (unsigned long long)(z == 123.456f);
                // online softmax (base 2)
                const float m_new = fmaxf(m_run, warp_max(z));
                const float corr = (m_run == -CUDART_INF_F) ? 0.f : exp2f((m_run - m_new) * LOG2E_F);
                // (TOK: a masked row is -inf, and so may be m_new for a tile with no visible row: its p must be 0, not NaN)
                const float pj = (lane < nrows && (!TOK || z != -CUDART_INF_F)) ? exp2f((z - m_new) * LOG2E_F) : 0.f;
                l_run = l_run * corr + pj;   // per-LANE partial sum (corr is warp-uniform): reduced once, before the state is stored
                m_run = m_new;
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[i] *= corr;
                if (DBG && wrec) wrec[12] = clk64() + (unsigned long long)(pj == 123.456f);
                // o += p_r * V_r on the FP32 pipe: lane owns 4 dims, 4 rows in flight
                {
                    const uint8_t *vbase = slots + (KREG ? 0 : D * 2) + lane * 8;
                    int rr = 0;
                    for (; rr + 4 <= nrows; rr += 4) {
                        uint2 vv[4];
                        float pv[4];
#pragma unroll
                        for (int uu = 0; uu < 4; ++uu) {
                            vv[uu] = *reinterpret_cast<const uint2 *>(vbase + (size_t)(rr + uu) * SSTRIDE);
                            pv[uu] = __shfl_sync(0xffffffffu, pj, rr + uu);
                        }
#pragma unroll
                        for (int uu = 0; uu < 4; ++uu) {
                            ffma2(acc[0], acc[1], pv[uu], bf16lo(vv[uu].x), bf16hi(vv[uu].x));
                            ffma2(acc[2], acc[3], pv[uu], bf16lo(vv[uu].y), bf16hi(vv[uu].y));
                        }
                    }
                    for (; rr < nrows; ++rr) {
                        const uint2 v = *reinterpret_cast<const uint2 *>(vbase + (size_t)rr * SSTRIDE);
                        const float pv = __shfl_sync(0xffffffffu, pj, rr);
                        ffma2(acc[0], acc[1], pv, bf16lo(v.x), bf16hi(v.x));
                        ffma2(acc[2], acc[3], pv, bf16lo(v.y), bf16hi(v.y));
                    }
                }
                __syncwarp();
                if (j + ncw_eff < ntile || base + selcap < tot) fence_proxy_async();  // this tile's generic-proxy reads precede the next tile's async-proxy writes
                if (DBG && !KREG) {
                    if (p.dbg && lane == 0 && j == warp && blockIdx.x < 16 && base == 0 &&
                        gridDim.x + blockIdx.x * 32 + warp < (unsigned)p.dbg_cap)
                        p.dbg[((size_t)(gridDim.x + blockIdx.x * 32 + warp)) * 16 + 6] = clk64();   // tile computed
                }
            }
        }
        if (base + selcap < tot) __syncthreads();   // the list (and the scan scratch) is rewritten by the next pass
    }
    if (DBG) t_dbg[7] = clk64();

    // ---- P6: MERGE -- warps -> CTA (shared memory) -> rank 0 of the cluster (distributed shared memory) ----------------
    // a warp's state goes to the start of its own (now idle) row buffer
    if (warp < ncw_eff) store_state(reinterpret_cast<float *>(slots), m_run, warp_sum(l_run), acc, lane);
    __syncthreads();
    // warps -> CTA: four warps, one output dimension per lane (a single warp needed ~1.4 us for 26 states: ~200 dependent
    // instructions with nothing else running).  Same products as merge_states, summed in two interleaved chains.
    if (warp < 4) {
        auto slot_ptr = [&](int i) {
            return (const float *)((i < ncw) ? slots_all + (size_t)i * FT * SSTRIDE : smem_raw + (size_t)(i - ncw) * FT * SSTRIDE);
        };
        unsigned long long t_rel = 0;
        float m_i = -CUDART_INF_F, l_i = 0.f;
        if (lane < ncw_eff) {
            const float *pp = slot_ptr(lane);
            m_i = pp[0];
            l_i = pp[1];
        }
        if (DBG) t_rel = clk64() + (unsigned long long)(m_i == 123.456f);   // barrier RELEASED (the read depends on it)
        const float mn = warp_max(m_i);
        const float f_i = (m_i == -CUDART_INF_F) ? 0.f : exp2f((m_i - mn) * LOG2E_F);
        const int dd = warp * 32 + lane;
        float a = 0.f, a_odd = 0.f;   // two accumulation chains (even / odd states)
#pragma unroll 4
        for (int i = 0; i + 1 < ncw_eff; i += 2) {
            a = fmaf(slot_ptr(i)[4 + dd], __shfl_sync(0xffffffffu, f_i, i), a);
            a_odd = fmaf(slot_ptr(i + 1)[4 + dd], __shfl_sync(0xffffffffu, f_i, i + 1), a_odd);
        }
        if (ncw_eff & 1) a = fmaf(slot_ptr(ncw_eff - 1)[4 + dd], __shfl_sync(0xffffffffu, f_i, ncw_eff - 1), a);
        a += a_odd;
        // CTA state -> slot c of rank 0:  m, l, count | acc[128]
        float *dst = s_cpart + (size_t)c * PART_FLOATS;
        st_shared_cluster_u32(dst + 4 + dd, 0, __float_as_uint(a));
        if (warp == 0) {
            const float L_ = warp_sum(l_i * f_i);
            if (lane == 0) st_shared_cluster_f4(dst, 0, make_float4(mn, L_, __int_as_float(tot), 0.f));
            if (DBG && p.dbg && lane == 0 && blockIdx.x < 16 && gridDim.x + blockIdx.x * 32 + 31 < (unsigned)p.dbg_cap) {
                unsigned long long *wr = p.dbg + ((size_t)(gridDim.x + blockIdx.x * 32 + 31)) * 16;   // record of warp 31 (never has a tile)
                wr[0] = t_rel;
                wr[1] = clk64() + (unsigned long long)(a == 123.456f);   // CTA state merged
                wr[5] = t_dbg[6];
            }
        }
    }
    if (p.results_out && tid == 0)
        for (unsigned rr = 0; rr < C; ++rr) st_shared_cluster_u32(&s_counts[c], rr, (uint32_t)tot);
    if (DBG) t_dbg[8] = clk64();
    cluster_barrier();
    if (c == 0 && warp == 0) {
        float M_, L_, A[4];
        merge_states<false>([&](int i) { return (const float *)(s_cpart + (size_t)i * PART_FLOATS); }, (int)C, lane, M_, L_, A);
        // softmax_kernel :238-239 (base-2 LSE) + wv_kernel :345 (fp32 -> bf16, FBGEMM rounding)
        const float inv = (L_ > 0.f) ? 1.0f / L_ : 0.f;
        const float o0 = A[0] * inv, o1 = A[1] * inv, o2 = A[2] * inv, o3 = A[3] * inv;
        const uint32_t lo = (uint32_t)f32_to_bf16_half_up(o0) | ((uint32_t)f32_to_bf16_half_up(o1) << 16);
        const uint32_t hi = (uint32_t)f32_to_bf16_half_up(o2) | ((uint32_t)f32_to_bf16_half_up(o3) << 16);
        *reinterpret_cast<uint2 *>(reinterpret_cast<uint8_t *>(p.out) + ((size_t)h * D + 4 * lane) * 2) = make_uint2(lo, hi);
        if (p.out_f32) *reinterpret_cast<float4 *>(p.out_f32 + (size_t)h * D + 4 * lane) = make_float4(o0, o1, o2, o3);
        if (p.peer_blocks) {
            // tensor-parallel epilogue (SURVEY 8 f3; replaces the per-layer all-gather of llama_dist-style TP): this head's
            // 256-byte row goes straight into every rank's gather slot over NVLink as 32 flag-carrying 16-byte lines (peer.cu:
            // {word, flag, word, flag}) -- no fence, no atomic; the consumer polls the lines
            const unsigned long long ep = p.peer_local[16];
            const int parity = (int)((ep + 1ull) & 1ull);
            const uint32_t flag = (uint32_t)(ep + 1ull);
            for (int rr = 0; rr < p.peer_world; ++rr) {
                uint8_t *slot = p.peer_blocks[rr] + ((size_t)parity * p.peer_world + p.peer_rank) * 2 * p.peer_slot_bytes;
                uint4 *line = reinterpret_cast<uint4 *>(slot) + (size_t)h * (D / 4) + lane;
                asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(line), "r"(lo), "r"(flag), "r"(hi), "r"(flag) : "memory");
            }
        }
        if (p.host_flags) {   // the host spins on these instead of paying a stream synchronisation
            __threadfence_system();
            __syncwarp();
            if (lane == 0) p.host_flags[h] = p.host_epoch;
        }
        if (lane == 0) {
            if (p.mve) {
                const float mv = M_ * LOG2E_F;
                p.mve[h] = mv;
                p.mve[p.H + h] = (L_ > 0.f) ? log2f(L_) + mv : -CUDART_INF_F;
            }
            int total_all = 0;
            for (unsigned rr = 0; rr < C; ++rr) total_all += __float_as_int(s_cpart[(size_t)rr * PART_FLOATS + 2]);
            p.nnz_out[h] = total_all;
        }
    }
    // optional outputs for mpig_last_probe / mpig_lsh_get_mask: the ascending index list and the collision bitmaps
    if (p.results_out) {
        int basep = 0;
        for (unsigned rr = 0; rr < c; ++rr) basep += s_counts[rr];
        int32_t *res = p.results_out + (size_t)h * M + basep;
        int tot2;
        const int cnt2 = select_count();
        const int pp0 = block_exclusive_scan_1bar(cnt2, wsum, &tot2);
        if (cnt2 > 0) select_emit(pp0, [&](int pp, int key) { res[pp] = lo_key + key; });
    }
    if (p.bitmaps_out) {
        uint32_t *bo = p.bitmaps_out + (size_t)h * 2 * p.words;
        for (int w = tid; w < Mc / 32; w += THREADS) {
            const int gw = lo_key / 32 + w;
            if (gw >= p.words || lo_rel + w * 32 >= p.seg_len) break;   // ranges are padded to 32 keys: stay inside this CTA's segment
            uint32_t b1 = 0, b2 = 0;
            for (int b = 0; b < 32; ++b) {
                const TagT v = tag[w * 32 + b];
                b1 |= (uint32_t)(v != EMPTY) << b;
                b2 |= (uint32_t)(v == SEL) << b;
            }
            bo[gw] = b1;
            bo[p.words + gw] = b2;
        }
    }
    if (DBG && p.dbg && tid == 0) {
        t_dbg[9] = clk64();
        t_dbg[10] = (unsigned long long)tot;
        t_dbg[11] = (unsigned long long)total_chunks;
#pragma unroll
        if (blockIdx.x < (unsigned)p.dbg_cap)
            for (int i = 0; i < 12; ++i) p.dbg[(size_t)blockIdx.x * 16 + i] = t_dbg[i];
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
struct FusedPlan {
    bool ok;
    ProbeGeom gm;
    int ncw;
    int threads;       // 1024 (one CTA per SM) or 512 (two)
    size_t smem;
    bool hash_in_kernel;
    FusedSmem lay;
    int cluster_waves;  // waves of clusters the grid needs (cudaOccupancyMaxActiveClusters; 0 = unknown)
};

using FusedKernel = void (*)(const FusedParams, const int32_t *, const int32_t *, const uint32_t *, const int32_t *);

// The fused_decode_kernel instantiation of a launch.  The T-token instantiations (tok) have no debug-clock variant; every variant
// has a shared spill twin (spill).
template <int THREADS, bool SPILL> static FusedKernel fused_kernel_of(bool dbg, bool kreg, bool tok) {
    if (tok) return kreg ? fused_decode_kernel<uint8_t, THREADS, false, true, true, SPILL> : fused_decode_kernel<uint8_t, THREADS, false, false, true, SPILL>;
    if (dbg) return kreg ? fused_decode_kernel<uint8_t, THREADS, true, true, false, SPILL> : fused_decode_kernel<uint8_t, THREADS, true, false, false, SPILL>;
    return kreg ? fused_decode_kernel<uint8_t, THREADS, false, true, false, SPILL> : fused_decode_kernel<uint8_t, THREADS, false, false, false, SPILL>;
}
static FusedKernel fused_kernel(int threads, bool dbg, bool kreg, bool tok, bool spill = false) {
    if (spill) return threads == 1024 ? fused_kernel_of<1024, true>(dbg, kreg, tok) : fused_kernel_of<512, true>(dbg, kreg, tok);
    return threads == 1024 ? fused_kernel_of<1024, false>(dbg, kreg, tok) : fused_kernel_of<512, false>(dbg, kreg, tok);
}

// dynamic shared memory a CTA may use: per SM 228 KB, less the static parameter block and the 1 KB the system reserves per CTA
static int fused_smem_cap(int threads) { return threads == 1024 ? 227 * 1024 - 1024 : 228 * 1024 / 2 - 2048; }

// A grid of `clusters` clusters of the plan's C CTAs, with programmatic stream serialization when pdl.  attr[2] backs cfg.attrs.
static cudaLaunchConfig_t fused_config(const FusedPlan &fp, int clusters, bool pdl, cudaStream_t s, cudaLaunchAttribute *attr) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(clusters * fp.gm.C);
    cfg.blockDim = dim3(fp.threads);
    cfg.dynamicSmemBytes = fp.smem;
    cfg.stream = s;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = fp.gm.C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 2 : 1;
    return cfg;
}

// Clusters of this plan's variant that the device keeps resident at once.  A cluster occupies SMs of ONE GPC, and the
// H100's GPCs have unequal SM counts, so #SMs / C over-counts; the runtime knows the real number.
static int fused_max_active_clusters(const FusedPlan &fp, bool kreg, bool tok, bool spill) {
    const FusedKernel fn = fused_kernel(fp.threads, false, kreg, tok, spill);
    if (func_attr_once((const void *)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, fused_smem_cap(fp.threads)) != MPIG_OK) return 0;
    cudaLaunchAttribute attr[2];
    const cudaLaunchConfig_t cfg = fused_config(fp, 1, false, 0, attr);
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, (const void *)fn, &cfg) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

// T > 1: the plan of the T-token instantiation for B*T*Hq virtual heads.  The segment geometry (and with it the cluster size C)
// was fixed at creation for B*Hq heads, so here B*T*Hq clusters may need several waves; they are independent of each other.
static FusedPlan fused_plan_compute(const mpig_ctx *ctx, int T = 1) {
    FusedPlan fp = {};
    fp.gm = probe_geometry(ctx);
    const int L = ctx->cfg.L, K = ctx->cfg.K;
    const int HT = ctx->H * T;
    if (L > 4 * 253) return fp;                              // one-byte tags: at most four passes of 253 tables
    if ((long long)L * ctx->cfg.max_length >= (1ll << 31)) return fp;   // chunk records hold 32-bit item offsets
    if (fp.gm.Sp > 8) return fp;
    // one wave of 1024-thread CTAs (one per SM), or 512-thread CTAs, two per SM: one wave up to 2 x #SMs CTAs, several waves
    // beyond that (large batches: one CTA per head, the CTAs are independent of each other)
    if (T == 1 && ctx->H * fp.gm.C > 2 * ctx->num_sms && fp.gm.C > 1) return fp;
    fp.threads = (HT * fp.gm.C > ctx->num_sms) ? 512 : 1024;
    // per CTA: dynamic + static (parameter block) + 1 KB the system reserves, out of 228 KB per SM
    const size_t cap = fused_smem_cap(fp.threads);
    const int stride = ctx->fused_kreg ? VSLOT : SLOT;
    const int max_warps = fp.threads / 32;
    int ncw = max_warps;
    for (; ncw >= 2; --ncw)
        if (fused_smem(fp.gm.Mc, 1, L, K, fp.gm.C, ncw, max_warps, ctx->fused_selcap, stride).total <= cap) break;
    if (ncw < 2) return fp;
    if ((((fp.gm.Mc / 4) + fp.threads - 1) / fp.threads | 1) > 31) return fp;   // a thread's run of tag words must fit two 64-bit masks
    fp.ncw = ncw;
    fp.lay = fused_smem(fp.gm.Mc, 1, L, K, fp.gm.C, ncw, max_warps, ctx->fused_selcap, stride);
    fp.smem = fp.lay.total;
    // the cluster splits the tables; with one CTA per head (large batches) every CTA would stream all of hash_func from L2:
    // those shapes hash in the separate tensor-core kernel (simhash.cu) and hand the codes over
    fp.hash_in_kernel = fp.gm.C >= 2;
    const int act = fused_max_active_clusters(fp, ctx->fused_kreg, T > 1, ctx->shared_spill);
    fp.cluster_waves = act > 0 ? (HT + act - 1) / act : 0;
    fp.ok = true;
    return fp;
}

// The plan depends on the (immutable) configuration, two options and the step size T: computed once per T (1..8), kept in the
// context.
static const FusedPlan &fused_plan(const mpig_ctx *ctx, int T = 1) {
    mpig_ctx *c = const_cast<mpig_ctx *>(ctx);
    const long long key = ((long long)ctx->fused_selcap << 8) | (ctx->fused_kreg ? 3 : 2);
    if (!c->fused_plan_cache) {
        c->fused_plan_cache = calloc(9, sizeof(FusedPlan));
        for (auto &k : c->fused_plan_key) k = 0;
    }
    if (!c->fused_plan_cache) {   // out of host memory: compute every time
        static thread_local FusedPlan tmp;
        tmp = fused_plan_compute(ctx, T);
        return tmp;
    }
    FusedPlan *fp = static_cast<FusedPlan *>(c->fused_plan_cache) + T;
    if (c->fused_plan_key[T] != key) {
        *fp = fused_plan_compute(ctx, T);
        c->fused_plan_key[T] = key;
    }
    return *fp;
}

bool fused_applicable(const mpig_ctx *ctx) { return ctx->decode_impl == 1 && fused_plan(ctx).ok; }
int fused_resident_clusters(int C, int threads) {
    FusedPlan fp = {};
    fp.gm.C = C;
    fp.threads = threads;
    fp.smem = fused_smem_cap(threads);   // the full carve-up the plan may use
    return fused_max_active_clusters(fp, false, false, false);
}
int fused_cluster_waves(const mpig_ctx *ctx) { return fused_plan(ctx).ok ? fused_plan(ctx).cluster_waves : 0; }

// The parameter block of a launch over the B*T*Hq (virtual) heads of T tokens per request; k / v = null: the rows were appended
// before the launch.  Left zero here: the debug buffer, the host flags and the peer exchange (single-token launches set them) and
// ntok (set by T-token launches).
static FusedParams fused_params(const mpig_ctx *ctx, int layer, const FusedPlan &fp, int T, const void *q, const void *k,
                                const void *v, void *out) {
    const LayerStore &ls = ctx->layers[layer];
    FusedParams p = {};
    p.q = (const __nv_bfloat16 *)q;
    p.k_new = (const __nv_bfloat16 *)k;
    p.v_new = (const __nv_bfloat16 *)v;
    p.avg_k = ls.avg_k;
    p.hf_t = ctx->hash_func_t;
    p.codes_in = fp.hash_in_kernel ? nullptr : ctx->codes;
    p.offsets = ls.offsets;
    p.items = reinterpret_cast<const uint16_t *>(ls.items);
    p.kv = ls.kv;
    p.kn = ls.kn;
    p.win = ctx->Wcap > 0 ? ls.win : nullptr;
    p.win_len = ctx->win_len;
    p.out = (__nv_bfloat16 *)out;
    p.out_f32 = ctx->want_out_f32 ? ctx->out_f32 : nullptr;
    p.mve = ctx->mve;
    p.nnz_out = ctx->nnz;
    p.results_out = ctx->save_mask ? ctx->results : nullptr;   // the index list goes to HBM only on request
    p.bitmaps_out = ctx->save_mask ? ctx->bitmaps : nullptr;
    p.codes_out = (ctx->save_mask && fp.hash_in_kernel) ? ctx->codes : nullptr;
    p.issue_win = ctx->fused_issue_win;
    p.H = ctx->H * T;
    p.G = ctx->G;
    p.Hq = ctx->cfg.num_attention_heads;
    p.M = ctx->cfg.max_length;
    p.Wcap = ctx->Wcap;
    p.K = ctx->cfg.K;
    p.L = ctx->cfg.L;
    p.NB = ctx->NB;
    p.S = ctx->nseg;
    p.r = fp.gm.r;
    p.Mc = fp.gm.Mc;
    p.words = ctx->bitmap_words;
    p.ncw = fp.ncw;
    p.selcap = ctx->fused_selcap;
    p.C = fp.gm.C;
    p.seg_len = ctx->seg_len;
    p.lay = fp.lay;
    return p;
}

// One launch over p.H clusters.  The instantiation follows from the block: the debug-clock one when p.dbg is set, the T-token
// one (with the pending step's ancestor masks, plan_kernel) when p.ntok is.
static int fused_launch(mpig_ctx *ctx, int layer, const FusedPlan &fp, const FusedParams &p, bool pdl, cudaStream_t s) {
    const bool tok = p.ntok > 0;
    const FusedKernel fn = fused_kernel(fp.threads, p.dbg != nullptr, ctx->fused_kreg, tok, ctx->shared_spill);
    MPIG_FUNC_ATTR(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, fused_smem_cap(fp.threads));
    cudaLaunchAttribute attr[2];
    const cudaLaunchConfig_t cfg = fused_config(fp, p.H, pdl, s, attr);
    const int32_t *anc = tok ? step_masks(ctx->step_buf) : nullptr;
    MPIG_CUDA(cudaLaunchKernelEx(&cfg, fn, p, anc, ctx->slot_map(), ctx->vis_map(), ctx->private_lo_map(layer)));
    MPIG_LAUNCH_CHECK(ctx);
    ctx->last_decode_fused = 1;
    return MPIG_OK;
}

void peer_epilogue_view(const mpig_peer *p, uint8_t *const **blocks, unsigned long long **local, size_t *slot_bytes, size_t *data_bytes);

int launch_fused(mpig_ctx *ctx, int layer, const void *q, const void *k, const void *v, void *out, cudaStream_t s, bool pdl,
                 const mpig_peer *peer, int peer_rank, int peer_world, volatile uint32_t *host_flags, uint32_t host_epoch) {
    const FusedPlan &fp = fused_plan(ctx);
    MPIG_REQUIRE(fp.ok, MPIG_EUNSUPPORTED, "fused decode: shape not supported (L=%d, H=%d, segments=%d)", ctx->cfg.L, ctx->H, ctx->nseg);
    if (!fp.hash_in_kernel) {
        int rc = launch_simhash(ctx, q, ctx->codes, ctx->qnorm, nullptr, s, pdl && ctx->pdl_first);
        if (rc) return rc;
    } else {
        MPIG_REQUIRE(ctx->hash_func_set, MPIG_ESTATE, "SimHash before mpig_set_hash_func: the projection has not been set");
    }
    FusedParams p = fused_params(ctx, layer, fp, 1, q, k, v, out);
    p.dbg = ctx->fused_debug ? ctx->fused_dbg : nullptr;
    p.dbg_cap = ctx->num_sms * 8;
    p.host_flags = host_flags;
    p.host_epoch = host_epoch;
    if (peer) {
        unsigned long long *loc = nullptr;
        peer_epilogue_view(peer, &p.peer_blocks, &loc, &p.peer_slot_bytes, &p.peer_data_bytes);
        p.peer_local = loc;
        p.peer_rank = peer_rank;
        p.peer_world = peer_world;
    }
    const int rc = fused_launch(ctx, layer, fp, p, pdl && (ctx->pdl_first || !fp.hash_in_kernel), s);
    if (rc) return rc;
    ctx->last_tokens = 1;
    ctx->last_chunk = false;
    return MPIG_OK;
}

int launch_fused_tokens(mpig_ctx *ctx, int layer, int T, const void *q, const void *k, const void *v, void *out, cudaStream_t s) {
    MPIG_REQUIRE(ctx->decode_impl == 1, MPIG_EUNSUPPORTED, "mpig_decode_tokens: T=%d needs the fused decode (decode_impl = 1)", T);
    const FusedPlan &fp = fused_plan(ctx, T);
    MPIG_REQUIRE(fp.ok, MPIG_EUNSUPPORTED, "mpig_decode_tokens: shape not supported by the fused decode (L=%d, H=%d, T=%d, segments=%d)",
                 ctx->cfg.L, ctx->H, T, ctx->nseg);
    MPIG_REQUIRE(ctx->hash_func_set, MPIG_ESTATE, "SimHash before mpig_set_hash_func: the projection has not been set");
    int rc = MPIG_OK;
    if (ctx->Wcap > 0) {   // the T new rows (centred keys) go to the window first: the attention reads them from HBM
        rc = launch_append_tokens(ctx, append_params(ctx, ctx->layers[layer], k, v, false), T, s);
        if (rc) return rc;
    }
    if (!fp.hash_in_kernel) {
        // one CTA per virtual head: the B*T*Hq query rows are hashed by the stand-alone tensor-core kernel
        rc = launch_simhash(ctx, q, ctx->codes, ctx->qnorm, nullptr, s, true, ctx->H * T);
        if (rc) return rc;
    }
    FusedParams p = fused_params(ctx, layer, fp, T, q, nullptr, nullptr, out);
    p.ntok = T;
    rc = fused_launch(ctx, layer, fp, p, true, s);   // under PDL behind the append (or the SimHash kernel)
    if (rc) return rc;
    ctx->last_tokens = T;
    ctx->last_chunk = false;
    ctx->last_tokens_waves = fp.cluster_waves;
    return MPIG_OK;
}

}  // namespace mpig
