// attend_dense.cu -- dense layers (models/attnserver.py:235-259): plain softmax attention of every q-head over the whole
// context (prefill rows + generated rows), the part the reference hands to FlashInfer's paged decode.
//
// Unlike the sampled layers, all G q-heads of a kv-group read the SAME rows, so the kernel is organised per
// (request, kv-head) group: each fetched 512-byte K|V record is used for all T*G <= 32 query rows of the group (G heads for
// each of the step's T tokens), i.e. HBM and L2 see every record once (the generic gather kernel in range mode fetched it G
// times and was L2-bound), and dense KV bytes per step do not grow with T.  Query rows sit on the M axis of the tensor-core
// tiles:
//     S^T (rows x 32 keys) = Q_g (16 x 128) . K_tile^T      A = Q fragments (registers), B = K rows (ldmatrix)
//     O   (rows x 128)    += P (16 x 32) . V_tile           P as bf16(p) + bf16(p - bf16(p))
// so the score accumulators of one lane are exactly the A fragment of the second product (no shuffles).
// Work decomposition, fetch (one cp.async.bulk per row, 528-byte slots) and the two-level last-arriver merge are the
// ones of attend_mma.cu with "kv-group" in place of "head".
#include "attend_common.cuh"

namespace mpig {

struct DenseParams {
    const uint8_t *kv;       // [BG][M] records
    const int32_t *len;      // [B]
    const __nv_bfloat16 *q;  // [B][T][Hq][D]
    __nv_bfloat16 *out;      // [B][T][Hq][D]
    float *out_f32;          // [B][T][Hq][D] or null: the output before the bf16 rounding (option "out_f32")
    float *partials;         // [grid][2][query rows per group][PART_FLOATS]
    int32_t *counters;       // [BG]
    int BG, G, Hkv, Hq, M;
};

__device__ __forceinline__ void finalize_dense_head(const DenseParams &p, int h, float l, const float acc[4], int lane) {
    __nv_bfloat16 *out = p.out;
    const float inv = (l > 0.f) ? 1.0f / l : 0.f;
    if (p.out_f32)
        *reinterpret_cast<float4 *>(p.out_f32 + (size_t)h * D + 4 * lane) = make_float4(acc[0] * inv, acc[1] * inv, acc[2] * inv, acc[3] * inv);
    uint32_t lo = (uint32_t)f32_to_bf16_half_up(acc[0] * inv) | ((uint32_t)f32_to_bf16_half_up(acc[1] * inv) << 16);
    uint32_t hi = (uint32_t)f32_to_bf16_half_up(acc[2] * inv) | ((uint32_t)f32_to_bf16_half_up(acc[3] * inv) << 16);
    *reinterpret_cast<uint2 *>(reinterpret_cast<uint8_t *>(out) + ((size_t)h * D + 4 * lane) * 2) = make_uint2(lo, hi);
}

// Partition of the groups' rows over the nw warps of the grid (one warp runs it): s_prefix[bg] = first row of group bg in the
// concatenation of all groups' rows, s_wpre[bg] = its first work item; a group of t rows gets max(1, t / Rp) items of >= TILE
// rows, so the items number at most nw whenever nw > BG (a warp then takes at most one item).  rows_of(bg) = the rows of group bg
// of the BG groups.
template <class RowsOf>
__device__ __forceinline__ void dense_partition_of(RowsOf rows_of, int BG, int *s_prefix, int *s_wpre, int nw, int lane) {
    int run = 0;
    for (int g0 = 0; g0 < BG; g0 += 32) {
        const int bg = g0 + lane;
        const int t = (bg < BG) ? rows_of(bg) : 0;
        int inc = t;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        if (bg < BG) s_prefix[bg] = run + inc - t;
        run += __shfl_sync(0xffffffffu, inc, 31);
    }
    const int total = run;
    if (lane == 0) s_prefix[BG] = total;
    const int Rp = (nw > BG) ? max(TILE, (total + (nw - BG) - 1) / (nw - BG)) : 0x3fffffff;
    __syncwarp();
    run = 0;
    for (int g0 = 0; g0 < BG; g0 += 32) {
        const int bg = g0 + lane;
        int w = 0;
        if (bg < BG) {
            const int t = s_prefix[bg + 1] - s_prefix[bg];
            w = (t > 0) ? max(1, t / Rp) : 0;
        }
        int inc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        if (bg < BG) s_wpre[bg] = run + inc - w;
        run += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) s_wpre[BG] = run;
}

// the group work item `item` belongs to (s_wpre ascending)
__device__ __forceinline__ int dense_item_group(const int *s_wpre, int BG, int item) {
    int a = 0, b = BG;
    while (b - a > 1) {
        const int mid = (a + b) >> 1;
        if (s_wpre[mid] <= item) a = mid; else b = mid;
    }
    while (s_wpre[a + 1] <= item) ++a;
    return a;
}

// ---- query rows, masks, merge ------------------------------------------------------------------------------------------------
// Row r = t*G + j of a group is q-head j of the group for token t; the rows sit on the M axis of NMT m16 tiles.  Token t sees the
// rows [0, len - T) before the step and those of the step's rows len - T + j whose bit j is set in its ancestor mask anc[b*T + t]
// (plan_kernel; a chain sets bits 0..t, i.e. rows [0, len - (T-1-t)): causal).  anc = null is a single-token decode: the step row
// is visible, and the step buffer is not read.
//   PACK (T*G <= 8): one m-tile whose rows 8..15 are free carry the lo halves of the bf16 hi/lo split of P;
//   otherwise the lo halves are a second pass of MMAs over each m-tile into the same accumulators.
// States of the T*G rows fill a warp's whole ring (32 x 132 floats at T*G = 32): the CTA-level merge reads the other warps' rings in
// place.  That is safe because a warp whose group is split (w_g > 1) never takes a second item (see the partition: then the items
// number at most the warps).
//
// SLOTS (shared dense mode): a group is (chunk, kv-head) instead, where a chunk is up to sl.cm requests
// bound to one slot (dense_slot_chunks).  Its query rows are (member, t, j), member-major; its rows are the chunk's prefix in the
// slot store, read once for all members, then each member's tail.  Prefix row k is visible to a member when k < its base; a
// member's tail rows are visible to its own query rows only, the step rows among them by the ancestor mask as above.
struct DenseSlots {
    const int32_t *slot_of;  // [B] slot of each request
    const int32_t *base;     // [B] dense_base: first row of each request in its tail
    const uint8_t *tail;     // [BG][R] records
    int B, R, cm;            // cm = requests per chunk: max(1, 32 / (T*G))
};

// Shared dense mode, warp 0: the chunks.  s_order = the requests by (slot, index); chunk c holds positions [s_cstart[c],
// s_cstart[c + 1]) (at most sl.cm requests of one slot), s_cstart[B + 1] = the chunk count.  The rows of a chunk's group are its
// prefix [0, max s_pre) of the slot store, then each member's tail: member m (a position) sees the prefix rows below s_pre[m] =
// min(base, dense_len) and its tail at [s_tbeg[m], s_tend[m]), so the group has s_tend[last member] rows.  O(B^2 / 32)
// shared-memory reads per lane (B at B <= 32).
__device__ __forceinline__ void dense_slot_chunks(const DenseParams &p, const DenseSlots &sl, int *s_order, int *s_pre, int *s_tbeg,
                                                  int *s_tend, int *s_cstart, int lane) {
    const int B = sl.B;
    int *s_slot = s_tend, *s_first = s_tbeg;   // scratch until the last pass writes them
    for (int b = lane; b < B; b += 32) s_slot[b] = sl.slot_of[b];
    __syncwarp();
    for (int b = lane; b < B; b += 32) {
        const int sb = s_slot[b];
        int before = 0, rank = 0;
        for (int j = 0; j < B; ++j) {
            const int sj = s_slot[j];
            before += (sj < sb);
            rank += (sj == sb && j < b);
        }
        s_order[before + rank] = b;
        s_first[before + rank] = (rank % sl.cm == 0);
    }
    __syncwarp();
    int nc = 0;
    for (int m0 = 0; m0 < B; m0 += 32) {
        const int m = m0 + lane;
        const bool f = m < B && s_first[m];
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        if (f) s_cstart[nc + __popc(bal & ((1u << lane) - 1u))] = m;
        nc += __popc(bal);
    }
    __syncwarp();
    if (lane == 0) {
        s_cstart[nc] = B;
        s_cstart[B + 1] = nc;
    }
    __syncwarp();
    for (int c = lane; c < nc; c += 32) {
        const int cs = s_cstart[c], ce = s_cstart[c + 1];
        int pc = 0;
        for (int m = cs; m < ce; ++m) {
            const int b = s_order[m];
            s_pre[m] = min(max(min(sl.base[b], p.len[b]), 0), p.M);
            pc = max(pc, s_pre[m]);
        }
        for (int m = cs; m < ce; ++m) {
            const int b = s_order[m];
            s_tbeg[m] = pc;
            pc += min(max(p.len[b] - sl.base[b], 0), sl.R);
            s_tend[m] = pc;
        }
    }
}

// smem: ring [warps][32][528] (reused as merge scratch once a warp's rows are done) | bars [warps] u64 | s_cnt [warps]
//       | s_prefix [BG+1] | s_wpre [BG+1] | SLOTS: the chunks (below)
// Up to 384 threads for the packed default-layout instantiation, which single-token decode launches with 12 warps (168 registers);
// the other instantiations need more than the 168 registers a 384-thread bound allows, or spill under it.
template <int NMT, bool PACK, bool SLOTS>
__global__ void __launch_bounds__((PACK && !SLOTS) ? 384 : 256)
    attend_dense_kernel(const DenseParams p, int T, const int32_t *anc, const DenseSlots sl) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t *slots = smem + (size_t)warp * TILE * SLOT;
    uint8_t *sp = smem + (size_t)warps * TILE * SLOT;
    uint64_t *bar = reinterpret_cast<uint64_t *>(sp) + warp;
    sp += (size_t)warps * sizeof(uint64_t);
    int *s_cnt = reinterpret_cast<int *>(sp);
    sp += (size_t)warps * sizeof(int);
    int *s_prefix = reinterpret_cast<int *>(sp);
    int *s_wpre = s_prefix + p.BG + 1;
    // SLOTS: s_order [B] | s_pre [B] | s_tbeg [B] | s_tend [B] | s_cstart [B + 2] (dense_slot_chunks)
    int *s_order = s_wpre + p.BG + 1, *s_pre = s_order + sl.B, *s_tbeg = s_pre + sl.B, *s_tend = s_tbeg + sl.B, *s_cstart = s_tend + sl.B;
    float *s_own = reinterpret_cast<float *>(slots);
    auto s_part_of = [&](int w) { return reinterpret_cast<float *>(smem + (size_t)w * TILE * SLOT); };
    const int G = p.G, TG = T * G;
    const int QS = SLOTS ? sl.cm * TG : TG;   // query rows a group may have: the stride of its states in the partial scratch

    if (lane == 0) {
        mbar_init(bar, 1);
        fence_proxy_async();
    }
    if (threadIdx.x < warps) s_cnt[threadIdx.x] = 0;
    pdl_wait();

    const int nw = gridDim.x * warps;
    if (warp == 0) {
        if constexpr (SLOTS) {
            dense_slot_chunks(p, sl, s_order, s_pre, s_tbeg, s_tend, s_cstart, lane);
            __syncwarp();
            dense_partition_of([&](int g) { return s_tend[s_cstart[g / p.Hkv + 1] - 1]; }, s_cstart[sl.B + 1] * p.Hkv, s_prefix, s_wpre,
                               nw, lane);
        } else {
            dense_partition_of([&](int g) { return min(max(p.len[g / p.Hkv], 0), p.M); }, p.BG, s_prefix, s_wpre, nw, lane);
        }
    }
    __syncthreads();
    pdl_launch_dependents();

    const int NG = SLOTS ? s_cstart[sl.B + 1] * p.Hkv : p.BG;   // groups
    const int u = blockIdx.x * warps + warp;
    const int n_items = s_wpre[NG];
    const int cta_w0 = blockIdx.x * warps;
    // output row of query row r of group bg: (B, T, Hq) order
    auto out_row = [&](int bg, int r) {
        if constexpr (SLOTS) {
            const int rt = r % TG;
            return (s_order[s_cstart[bg / p.Hkv] + r / TG] * T + rt / G) * p.Hq + (bg % p.Hkv) * G + rt % G;
        } else {
            return ((bg / p.Hkv) * T + r / G) * p.Hq + (bg % p.Hkv) * G + r % G;
        }
    };
    // query rows of group bg
    auto rows_q = [&](int bg) { return SLOTS ? (s_cstart[bg / p.Hkv + 1] - s_cstart[bg / p.Hkv]) * TG : TG; };

    for (int bg = u; bg < NG; bg += nw) {
        if (s_prefix[bg + 1] == s_prefix[bg]) {
            const float z4[4] = {0.f, 0.f, 0.f, 0.f};
            for (int r = 0; r < rows_q(bg); ++r) finalize_dense_head(p, out_row(bg, r), 0.f, z4, lane);
        }
    }

    const float scale_log2 = rsqrtf((float)D) * LOG2E_F;
    const int grp = lane >> 2, tig = lane & 3;
    const uint32_t slots_s = smem_u32(slots);
    const uint32_t k_lane_off = (uint32_t)(((lane & 7) + (lane >> 4) * 8) * SLOT + ((lane >> 3) & 1) * 16);
    const uint32_t v_lane_off = (uint32_t)(((lane & 7) + ((lane >> 3) & 1) * 8) * SLOT + D * 2 + (lane >> 4) * 16);
    constexpr int NI = PACK ? 1 : 2;   // query rows a lane holds per m-tile: grp (and grp + 8)
    constexpr bool QREG = (NMT == 1);  // one m-tile: the q fragments stay in registers; two: re-read per tile (L1)
    // the instantiation single-token decode runs: output rows read from one lane each, tile visibility as a bitmask (a division by
    // G per row and a branch per score measurably slow it; the other instantiations keep the per-row and per-score forms, which
    // cost them fewer registers and spills)
    constexpr bool FAST = PACK && !SLOTS;
    uint32_t phase = 0;

    for (int item = u; item < n_items; item += nw) {
        const int bg = dense_item_group(s_wpre, NG, item);
        const int len = s_prefix[bg + 1] - s_prefix[bg];
        const int w_g = s_wpre[bg + 1] - s_wpre[bg];
        const int part = item - s_wpre[bg];
        const int c_g = (len + w_g - 1) / w_g;
        const int r_lo = part * c_g, r_hi = min(r_lo + c_g, len);
        const int qr = rows_q(bg);
        // FAST: lane r computes the output row of query row r, for the q rows below and the merge
        const int lane_row = FAST ? out_row(bg, min(lane, qr - 1)) : 0;
        // SLOTS: the chunk's first position, its prefix rows, and the slot store rows of this kv-head
        const int cs = SLOTS ? s_cstart[bg / p.Hkv] : 0, pc = SLOTS ? s_tbeg[cs] : 0;
        const uint8_t *rows = SLOTS ? p.kv + ((size_t)sl.slot_of[s_order[cs]] * p.Hkv + bg % p.Hkv) * p.M * REC
                                    : p.kv + (size_t)bg * p.M * REC;
        // the record of the group's row k
        auto row_src = [&](int k) {
            if constexpr (SLOTS) {
                if (k < pc) return rows + (size_t)k * REC;
                int m = cs;
                while (s_tend[m] <= k) ++m;
                return sl.tail + (((size_t)s_order[m] * p.Hkv + bg % p.Hkv) * sl.R + (k - s_tbeg[m])) * REC;
            } else {
                return rows + (size_t)k * REC;
            }
        };

        // this lane's query rows: r = mt*16 + i*8 + grp; rows past T*G are zero and unmasked.  Key row k is visible to query row r
        // when k < lim or bit k - lim of vis is set (lim = the first row of the step, vis = the token's ancestor mask); SLOTS: a
        // prefix row (k < pc) when k < pre, a tail row when that holds and k >= tb (the member's tail starts at tb)
        const uint32_t *qrow[NMT][2];
        int lim[NMT][2];
        uint32_t vis[NMT][2];
        int pre[SLOTS ? NMT : 1][2], tb[SLOTS ? NMT : 1][2];
#pragma unroll
        for (int mt = 0; mt < NMT; ++mt)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int r = mt * 16 + i * 8 + grp;
                const bool ok = r < qr && !(PACK && i == 1);
                const int row = FAST ? __shfl_sync(0xffffffffu, lane_row, r) : 0;
                qrow[mt][i] = ok ? reinterpret_cast<const uint32_t *>(p.q + (size_t)(FAST ? row : out_row(bg, r)) * D) : nullptr;
                if constexpr (SLOTS) {
                    const int m = cs + r / TG;   // the member's position (valid when ok)
                    lim[mt][i] = ok ? s_tend[m] - T : 0x3fffffff;
                    vis[mt][i] = ok ? (anc ? (uint32_t)__ldg(anc + s_order[m] * T + (r % TG) / G) : 1u) : 0u;
                    pre[mt][i] = ok ? s_pre[m] : 0x3fffffff;
                    tb[mt][i] = ok ? s_tbeg[m] : 0;
                } else {
                    lim[mt][i] = ok ? len - T : len;
                    vis[mt][i] = ok ? (anc ? (uint32_t)__ldg(anc + (bg / p.Hkv) * T + r / G) & ((1u << TREE_MAX) - 1u) : 1u) : 0u;
                }
            }
        auto q_frag = [&](int mt, int ks, uint32_t (&a)[4]) {
            a[0] = qrow[mt][0] ? __ldg(qrow[mt][0] + ks * 8 + tig) : 0u;
            a[1] = qrow[mt][1] ? __ldg(qrow[mt][1] + ks * 8 + tig) : 0u;
            a[2] = qrow[mt][0] ? __ldg(qrow[mt][0] + ks * 8 + 4 + tig) : 0u;
            a[3] = qrow[mt][1] ? __ldg(qrow[mt][1] + ks * 8 + 4 + tig) : 0u;
        };
        uint32_t qa[QREG ? 8 : 1][4];
        if (QREG) {
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) q_frag(0, ks, qa[QREG ? ks : 0]);
        }
        __syncwarp();
        fence_proxy_async();
        float m_run[NMT][2], l_run[NMT][2];
        float acc[NMT][16][4];
#pragma unroll
        for (int mt = 0; mt < NMT; ++mt) {
            m_run[mt][0] = m_run[mt][1] = -CUDART_INF_F;
            l_run[mt][0] = l_run[mt][1] = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[mt][i][0] = acc[mt][i][1] = acc[mt][i][2] = acc[mt][i][3] = 0.f;
        }

        for (int cr = r_lo; cr < r_hi; cr += TILE) {
            const int nrows = min(TILE, r_hi - cr);
            if (lane == 0) mbar_arrive_expect_tx(bar, (uint32_t)nrows * REC);
            __syncwarp();
            if (lane < nrows) {
                bulk_g2s(slots + (size_t)lane * SLOT, row_src(cr + lane), REC, bar);
            } else {
                uint4 *vz = reinterpret_cast<uint4 *>(slots + (size_t)lane * SLOT);
#pragma unroll
                for (int i = 0; i < 32; ++i) vz[i] = make_uint4(0, 0, 0, 0);
            }
            __syncwarp();
            mbar_wait(bar, phase);
            phase ^= 1;

            // ---- S^T = Q . K_tile^T per m-tile ----------------------------------------------------------------------
            float s[NMT][4][4];
#pragma unroll
            for (int mt = 0; mt < NMT; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) s[mt][nt][0] = s[mt][nt][1] = s[mt][nt][2] = s[mt][nt][3] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                uint32_t a[NMT][4];
#pragma unroll
                for (int mt = 0; mt < NMT; ++mt) {
                    if (QREG) {
                        a[mt][0] = qa[QREG ? ks : 0][0]; a[mt][1] = qa[QREG ? ks : 0][1];
                        a[mt][2] = qa[QREG ? ks : 0][2]; a[mt][3] = qa[QREG ? ks : 0][3];
                    } else {
                        q_frag(mt, ks, a[mt]);
                    }
                }
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    uint32_t b[4];
                    ldsm_x4(b, slots_s + (uint32_t)(j * 16 * SLOT + ks * 32) + k_lane_off);
#pragma unroll
                    for (int mt = 0; mt < NMT; ++mt) {
                        mma_16816(s[mt][2 * j], a[mt], b[0], b[1]);
                        mma_16816(s[mt][2 * j + 1], a[mt], b[2], b[3]);
                    }
                }
            }
            // ---- online softmax per query row (lane holds keys nt*8 + tig*2 + {0,1} of rows grp and grp+8) --------
            float corr[NMT][2];
#pragma unroll
            for (int mt = 0; mt < NMT; ++mt)
#pragma unroll
                for (int i = 0; i < NI; ++i) {
                    // FAST: bit r of `seen` = tile row r is visible, once per tile.  It must agree with the per-score rule
                    // below (key cr + r visible when r < nrows and (cr + r < lim or bit cr + r - lim of vis is set)).
                    uint32_t seen = 0;
                    if constexpr (FAST) {
                        const int o = lim[mt][i] - cr;   // tile row of the step's first row
                        seen = (o >= 32) ? ~0u : (o > 0 ? ~0u >> (32 - o) : 0u);
                        if (o > -TREE_MAX && o < 32) seen |= (o >= 0) ? vis[mt][i] << o : vis[mt][i] >> -o;
                        seen = (seen & (~0u >> (32 - nrows))) >> (tig * 2);
                    }
                    float mloc = -CUDART_INF_F;
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int r = nt * 8 + tig * 2 + e;
                            float &x = s[mt][nt][2 * i + e];
                            if constexpr (FAST) {
                                x = ((seen >> (nt * 8 + e)) & 1u) ? x * scale_log2 : -CUDART_INF_F;
                            } else {
                                const int o = cr + r - lim[mt][i];
                                bool vis_r = o < 0 || ((unsigned)o < (unsigned)TREE_MAX && ((vis[mt][i] >> o) & 1u));
                                if constexpr (SLOTS) vis_r = (cr + r < pc) ? (cr + r < pre[mt][i]) : (cr + r >= tb[mt][i] && vis_r);
                                x = (r < nrows && vis_r) ? x * scale_log2 : -CUDART_INF_F;
                            }
                            mloc = fmaxf(mloc, x);
                        }
                    mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 1));
                    mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 2));
                    const float m_new = fmaxf(m_run[mt][i], mloc);
                    const float m_use = (m_new == -CUDART_INF_F) ? 0.f : m_new;   // a row with no visible key yet: all p = 0
                    corr[mt][i] = (m_run[mt][i] == -CUDART_INF_F) ? 0.f : exp2f(m_run[mt][i] - m_new);
                    float lsum = 0.f;
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            float &x = s[mt][nt][2 * i + e];
                            x = exp2f(x - m_use);
                            lsum += x;
                        }
                    lsum += __shfl_xor_sync(0xffffffffu, lsum, 1);
                    lsum += __shfl_xor_sync(0xffffffffu, lsum, 2);
                    l_run[mt][i] = l_run[mt][i] * corr[mt][i] + lsum;
                    m_run[mt][i] = m_new;
                }
            if (cr > r_lo) {
#pragma unroll
                for (int mt = 0; mt < NMT; ++mt)
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        acc[mt][i][0] *= corr[mt][0]; acc[mt][i][1] *= corr[mt][0];
                        acc[mt][i][2] *= corr[mt][NI - 1]; acc[mt][i][3] *= corr[mt][NI - 1];
                    }
            }
            // ---- O += P . V (P as bf16 hi + lo) --------------------------------------------------------------------
            // (one m-tile at a time: its fragments only are live; the V fragments are re-read from shared memory per m-tile)
#pragma unroll
            for (int ks = 0; ks < 2; ++ks)
#pragma unroll
                for (int mt = 0; mt < NMT; ++mt) {
                    uint32_t ahi[4], alo[4];
#pragma unroll
                    for (int half = 0; half < 2; ++half)
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            // PACK: a[2*half] = hi of row grp, a[2*half+1] = lo of row grp (in row grp + 8)
                            const int src = PACK ? 0 : i;
                            const float p0 = s[mt][2 * ks + half][2 * src], p1 = s[mt][2 * ks + half][2 * src + 1];
                            const uint32_t h0 = f32_to_bf16_rne(p0), h1 = f32_to_bf16_rne(p1);
                            const uint32_t l0 = f32_to_bf16_rne(p0 - bf16_bits_to_f32(h0)), l1 = f32_to_bf16_rne(p1 - bf16_bits_to_f32(h1));
                            if (PACK) {
                                if (i == 0) ahi[2 * half] = h0 | (h1 << 16);
                                else ahi[2 * half + 1] = l0 | (l1 << 16);
                            } else {
                                ahi[2 * half + i] = h0 | (h1 << 16);
                                alo[2 * half + i] = l0 | (l1 << 16);
                            }
                        }
#pragma unroll
                    for (int n2 = 0; n2 < 8; ++n2) {
                        uint32_t b[4];
                        ldsm_x4_trans(b, slots_s + (uint32_t)(ks * 16 * SLOT + n2 * 32) + v_lane_off);
                        mma_16816(acc[mt][2 * n2], ahi, b[0], b[1]);
                        mma_16816(acc[mt][2 * n2 + 1], ahi, b[2], b[3]);
                        if (!PACK) {
                            mma_16816(acc[mt][2 * n2], alo, b[0], b[1]);
                            mma_16816(acc[mt][2 * n2 + 1], alo, b[2], b[3]);
                        }
                    }
                }
            __syncwarp();
            fence_proxy_async();
        }

        // ---- part done: states of the T*G rows -> [T*G][132] floats in the warp's idle ring -------------------------
        __syncwarp();
#pragma unroll
        for (int mt = 0; mt < NMT; ++mt)
#pragma unroll
            for (int i = 0; i < NI; ++i) {
                const int r = mt * 16 + i * 8 + grp;
                if (r < qr) {
                    float *st = s_own + (size_t)r * PART_FLOATS;
                    if (tig == 0) {
                        st[0] = m_run[mt][i] * 0.6931471805599453f;
                        st[1] = l_run[mt][i];
                    }
#pragma unroll
                    for (int nt = 0; nt < 16; ++nt) {
                        const float2 v = PACK ? make_float2(acc[mt][nt][0] + acc[mt][nt][2], acc[mt][nt][1] + acc[mt][nt][3])
                                              : make_float2(acc[mt][nt][2 * i], acc[mt][nt][2 * i + 1]);
                        *reinterpret_cast<float2 *>(st + 4 + nt * 8 + tig * 2) = v;
                    }
                }
            }
        __syncwarp();

        const int i0 = s_wpre[bg], i1 = i0 + w_g - 1;
        const int wa = max(i0, cta_w0), wb = min(i1, cta_w0 + warps - 1);
        bool carry = true;
        if (w_g > 1 && wb > wa) {
            // level 1: the states stay in each warp's ring; the last arriver of this CTA combines them
            int ticket = 0;
            if (lane == 0) ticket = atom_add_acq_rel_cta_shared(&s_cnt[wa - cta_w0], 1);
            ticket = __shfl_sync(0xffffffffu, ticket, 0);
            carry = (ticket == wb - wa);
        }
        if (!carry) continue;
        auto row_of = [&](int r) { return FAST ? __shfl_sync(0xffffffffu, lane_row, r) : out_row(bg, r); };
        const int cta_first = i0 / warps, cta_last = i1 / warps;
        const bool need_l1 = (w_g > 1 && wb > wa);
        const bool need_l2 = (w_g > 1 && cta_first != cta_last);
        int ticket2 = 0;
        float *gslot = p.partials + ((size_t)blockIdx.x * 2 + ((i0 >= cta_w0) ? 1 : 0)) * (size_t)QS * PART_FLOATS;
        for (int r = 0; r < qr; ++r) {
            float M_, L_, A[4];
            if (need_l1) {
                merge_states<false>([&](int i) { return (const float *)(s_part_of(wa - cta_w0 + i) + (size_t)r * PART_FLOATS); },
                                    wb - wa + 1, lane, M_, L_, A);
            } else {
                const float *st = s_own + (size_t)r * PART_FLOATS;
                M_ = st[0];
                L_ = st[1];
                const float4 o4 = *reinterpret_cast<const float4 *>(st + 4 + 4 * lane);
                A[0] = o4.x; A[1] = o4.y; A[2] = o4.z; A[3] = o4.w;
            }
            if (!need_l2) finalize_dense_head(p, row_of(r), L_, A, lane);
            else store_state(gslot + (size_t)r * PART_FLOATS, M_, L_, A, lane);
        }
        if (!need_l2) continue;
        __syncwarp();
        if (lane == 0) ticket2 = atom_add_acq_rel_gpu(p.counters + bg, 1);
        ticket2 = __shfl_sync(0xffffffffu, ticket2, 0);
        if (ticket2 == cta_last - cta_first) {
            for (int r = 0; r < qr; ++r) {
                float M_, L_, A[4];
                merge_states<true>(
                    [&](int i) {
                        const int c2 = cta_first + i;
                        return (const float *)(p.partials + ((size_t)c2 * 2 + ((i0 >= c2 * warps) ? 1 : 0)) * (size_t)QS * PART_FLOATS +
                                               (size_t)r * PART_FLOATS);
                    },
                    cta_last - cta_first + 1, lane, M_, L_, A);
                finalize_dense_head(p, row_of(r), L_, A, lane);
            }
            if (lane == 0) p.counters[bg] = 0;
        }
    }
}

int launch_attend_dense(mpig_ctx *ctx, const LayerStore &ls, int T, const void *q, void *out, cudaStream_t s, bool pdl) {
    const bool slots = ctx->dense_tail_rows > 0;
    const int B = ctx->cfg.batch_size, TG = T * ctx->G;
    DenseParams p = {};
    p.kv = ls.dense_kv;
    p.len = ctx->dense_len;
    p.q = (const __nv_bfloat16 *)q;
    p.out = (__nv_bfloat16 *)out;
    p.out_f32 = ctx->want_out_f32 ? ctx->out_f32 : nullptr;
    p.partials = ctx->partials;
    p.counters = ctx->counters;
    p.BG = ctx->BG;
    p.G = ctx->G;
    p.Hkv = ctx->cfg.num_key_value_heads;
    p.Hq = ctx->cfg.num_attention_heads;
    p.M = ctx->cfg.max_length;
    DenseSlots sl = {};
    if (slots) {
        sl.slot_of = ctx->slot_of;
        sl.base = ctx->dense_base;
        sl.tail = ls.dense_tail;
        sl.B = B;
        sl.R = ctx->dense_tail_rows;
        sl.cm = std::max(1, 32 / TG);
    }
    // the most query rows a group can have: T*G, or in slot mode a chunk of cm requests or all B bound to one slot (the bindings
    // may change after a capture, so the regime depends on B only); the partial scratch holds states of cm*T*G rows
    const int rows = slots ? std::min(sl.cm, B) * TG : TG;
    const int qs = slots ? sl.cm * TG : TG;
    // 12 warps for single-token decode in the default layout, 8 for every other launch: the warp count sets the row partition
    const int warps = (!slots && T == 1 && rows <= 8) ? 12 : 8;
    const size_t smem = (size_t)warps * (TILE * SLOT + 8 + 4) + 2 * (size_t)(p.BG + 1) * sizeof(int) +
                        (slots ? (size_t)(5 * B + 2) * sizeof(int) : 0) + 16;
    MPIG_REQUIRE(smem <= 227 * 1024, MPIG_EINVAL, "dense attention: %zu B shared memory", smem);
    // slot mode has at most B*Hkv groups (a chunk holds at least one request), so the counters suffice in both modes
    MPIG_REQUIRE((size_t)ctx->num_sms * 2 * qs <= (size_t)ctx->max_partial_warps * 2, MPIG_EINVAL, "dense attention: partial scratch too small");
    void (*kernel)(DenseParams, int, const int32_t *, DenseSlots);
    if (rows <= 8) kernel = slots ? attend_dense_kernel<1, true, true> : attend_dense_kernel<1, true, false>;
    else if (rows <= 16) kernel = slots ? attend_dense_kernel<1, false, true> : attend_dense_kernel<1, false, false>;
    else kernel = slots ? attend_dense_kernel<2, false, true> : attend_dense_kernel<2, false, false>;
    MPIG_FUNC_ATTR(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(ctx->num_sms);
    cfg.blockDim = dim3(warps * 32);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    const int32_t *anc = (T > 1) ? (const int32_t *)step_masks(ctx->step_buf) : nullptr;
    MPIG_CUDA(cudaLaunchKernelEx(&cfg, kernel, p, T, anc, sl));
    MPIG_LAUNCH_CHECK(ctx);
    ctx->last_tokens = T;
    ctx->last_chunk = false;
    return MPIG_OK;
}

}  // namespace mpig
