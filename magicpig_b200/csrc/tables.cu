// tables.cu -- HBM-resident LSH tables: build, and stage 2 (the probe).
//
// Replaces library/lsh/lsh.cc:
//   LSH::fill            :143-201  -> build_segments_kernel<true>  (same inputs: sorted codes + argsort)
//   sort()+LSH::fill     attnserver.py:186-193 -> build_segments_kernel<false> (counting sort on device)
//   LSH::batch_retrieve  :210-241, LSH::retrieve :243-288 -> probe_kernel
//   LSH::get_mask        :308-314  -> expand_mask_kernel
// and, with no reference equivalent, the table side of a window spill (mpig_spill_window, store.cu) -> table_merge_kernel, and
// of a compaction (mpig_compact_context, store.cu) -> table_truncate_kernel then table_merge_kernel
//
// Table format (per context slot c, kv-head g, table l; row = (c*Hkv+g)*L + l): segmented compact CSR.  Request b reads the tables
// of slot slot_of[b] (b itself when the map is null).
//   Keys are cut into S = ceil(M / 65536) segments of EQUAL length seg_len = ceil(M / S) rounded up to 64 (<= 65536; equal so
//   that the CTAs of a probing cluster own equal key ranges).  Segment s of a row owns the item region [s*seg_len, ...) of
//   items[row][0..M) (uint16 = key index - s*seg_len, grouped by bucket) and its own bucket starts
//   offsets[row][s][0..NB] (int32, absolute positions in the row): bucket c of segment s holds
//   items[row][offsets[row][s][c] .. offsets[row][s][c+1]).
// 2 bytes per (key, table) instead of the reference's 4 (lsh.h:40 `table`), which is what lets the ProLong config
// (n = 500K, L = 300: 2.4 GB instead of 4.8 GB per layer) keep 30 layers of tables beside the KV records in 180 GB,
// and a probing CTA reads only the sub-lists of the key segment it owns.
// The reference keeps table_start AND table_end (lsh.h:38-39); end[c] == start[c+1] once empty
// buckets are filled in, so one array of NB+1 entries carries the same information.
//
// Probe algorithm.  The reference walks the L buckets serially doing a read-modify-write of a 1-byte saturating counter
// per candidate in a 98 KB per-head mask (lsh.cc:272-283).  Here a thread-block CLUSTER owns one q-head; CTA c owns a key
// range inside one key segment and keeps one TAG per key of its range in shared memory, tag in {EMPTY, table id, SEL}
// <=> the reference's mask byte {0, 1, 2}.  The state machine is realised with two sweeps of plain, idempotent stores and no
// atomics: sweep 1 writes tag[key] = t for every candidate (table t, key); sweep 2 writes SEL wherever tag[key] != t.  A key
// hit by one table keeps that table's id; a key hit by >= 2 tables is marked by at least one loser of sweep 1.  All
// candidates of all L buckets are processed in parallel (32-candidate chunks, coalesced loads, the first chunks of a warp
// kept in registers between the sweeps), the tag array is swept once more to count and emit the SEL keys in ASCENDING order,
// and the CTAs of the cluster exchange their counts through distributed shared memory to place their pieces of the list.
#include "probe_common.cuh"

namespace mpig {

// ---------------------------------------------------------------------------------------------
// Table build: counting sort of one (kv-head, table, key segment) per CTA into the segmented compact layout.
//   SORTED = false  device route, replaces sort() + LSH::fill (attnserver.py:186-193): input = key codes (Hkv, L, n)
//   SORTED = true   LSH::fill itself (lsh.cc:143-201): input = sorted codes + argsort indices of the same shape; every
//                   CTA walks the whole sorted list and keeps the keys of its segment
// grid (L, Hkv, S), 1024 threads; dynamic smem = (NB + 1 + 40) ints [+ SEG uint16 staging when it fits].
// Order inside a bucket is unspecified (the probe does not depend on it).
// ---------------------------------------------------------------------------------------------
template <bool SORTED>
__global__ void __launch_bounds__(1024) build_segments_kernel(const int16_t *__restrict__ codes, const int32_t *__restrict__ idx,
                                                              int32_t *__restrict__ offsets, uint16_t *__restrict__ items, int n,
                                                              int NB, int M, int L, int S, int staged, int seg_len) {
    extern __shared__ int smem_i[];
    int *hist = smem_i;            // NB + 1
    int *wsum = smem_i + NB + 1;   // 33+
    uint16_t *stage = reinterpret_cast<uint16_t *>(wsum + 40);
    constexpr int T = 1024, UN = 8;
    const size_t row = (size_t)blockIdx.y * L + blockIdx.x;
    const int seg = blockIdx.z, tid = threadIdx.x;
    const int seg_lo = seg * seg_len;
    const int seg_hi = min(SORTED ? M : n, seg_lo + seg_len);   // keys [seg_lo, seg_hi) belong to this CTA
    const int16_t *c = codes + row * n;
    const int32_t *ix = SORTED ? idx + row * n : nullptr;
    int32_t *off = offsets + (row * S + seg) * (size_t)(NB + 1);
    uint16_t *it = items + row * (size_t)M + seg_lo;
    if (seg_lo >= seg_hi) {  // segment beyond the keys: every bucket empty
        for (int b = tid; b <= NB; b += T) off[b] = seg_lo;
        return;
    }
    for (int b = tid; b <= NB; b += T) hist[b] = 0;
    __syncthreads();
    // visits every (code, key) pair of this segment; loads are issued UN at a time so the pass is not one latency per element
    auto for_each_pair = [&](auto &&body) {
        if (!SORTED) {
            for (int k0 = seg_lo + tid; k0 < seg_hi; k0 += T * UN) {
                int cc[UN];
#pragma unroll
                for (int u = 0; u < UN; ++u) {
                    const int k = k0 + u * T;
                    cc[u] = (k < seg_hi) ? (int)c[k] : -1;
                }
#pragma unroll
                for (int u = 0; u < UN; ++u)
                    if (cc[u] >= 0 && cc[u] < NB) body(cc[u], k0 + u * T);
            }
        } else {
            for (int i0 = tid; i0 < n; i0 += T * UN) {
                int key[UN], cc[UN];
#pragma unroll
                for (int u = 0; u < UN; ++u) {
                    const int i = i0 + u * T;
                    key[u] = (i < n) ? ix[i] : -1;
                }
#pragma unroll
                for (int u = 0; u < UN; ++u) cc[u] = (key[u] >= seg_lo && key[u] < seg_hi) ? (int)c[i0 + u * T] : -1;
#pragma unroll
                for (int u = 0; u < UN; ++u)
                    if (cc[u] >= 0 && cc[u] < NB) body(cc[u], key[u]);
            }
        }
    };
    for_each_pair([&](int cc, int) { atomicAdd(&hist[cc], 1); });
    __syncthreads();
    // exclusive scan of hist[0..NB): thread t owns a contiguous chunk of bins
    const int per = (NB + T - 1) / T;
    const int b0 = tid * per, b1 = min(b0 + per, NB);
    int local = 0;
    for (int b = b0; b < b1; ++b) local += hist[b];
    int total;
    int base = block_exclusive_scan(local, wsum, &total);
    for (int b = b0; b < b1; ++b) {
        const int h = hist[b];
        hist[b] = base;             // becomes the running cursor (relative to the segment's item region)
        off[b] = seg_lo + base;     // absolute position in the row's item array
        base += h;
    }
    if (tid == 0) off[NB] = seg_lo + total;
    __syncthreads();
    if (staged) {
        for_each_pair([&](int cc, int key) { stage[atomicAdd(&hist[cc], 1)] = (uint16_t)(key - seg_lo); });
        __syncthreads();
        for (int j = tid; j < total; j += T) it[j] = stage[j];   // coalesced write-out
    } else {
        for_each_pair([&](int cc, int key) { it[atomicAdd(&hist[cc], 1)] = (uint16_t)(key - seg_lo); });
    }
}

// ---------------------------------------------------------------------------------------------
// Table merge of a window spill (mpig_spill_window): add the keys [n_old, n_old + g) of a context slot, whose codes are given,
// to its tables in place.  One CTA per (table, kv-head, slot x key segment), so no two CTAs write the same table row; segments
// the new keys do not touch return at once.
// With ex[c] = exclusive prefix of the histogram of the new codes over buckets and ro[c] = old offset relative to the segment:
//   new offset of bucket c           = ro[c] + ex[c]
//   old item at relative position p  -> p + ex[bucket(p)]          (old items of a bucket first ...)
//   new key of code c                -> ro[c + 1] + ex[c] + rank   (... then the new ones)
// The shift ex[bucket(p)] never decreases with p, so the old items are moved from the top of the segment down in chunks, each
// chunk read completely before any of it is written: a write lands only on positions already read.  No staging copy of the
// segment is needed, so every K works in place (the old offsets are kept in shared memory when they fit beside the
// histogram, K <= 14, and read from HBM otherwise).  A segment whose offsets are all equal has no old items, which covers a
// segment beyond the old keys and tables that were never built (offsets still zero).  grid (L, Hkv, C * S), 512 threads;
// dynamic smem = (NB + 1 + 40 [+ NB + 1 when staged]) ints.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512) table_merge_kernel(const int16_t *__restrict__ codes, int32_t *offsets, uint16_t *items,
                                                          const int32_t *__restrict__ spill_g, const int32_t *__restrict__ spill_pre,
                                                          const int32_t *__restrict__ spill_n_old, int Hkv, int L, int NB, int M, int S,
                                                          int seg_len, int staged) {
    extern __shared__ int smem_i[];
    constexpr int T = 512, UN = 4;
    int *ex = smem_i;                // NB + 1: histogram of the new codes -> exclusive prefix -> placement cursors
    int *wsum = smem_i + NB + 1;     // 40
    int *oo_s = wsum + 40;           // NB + 1 old offsets (staged)
    const int l = blockIdx.x, gi = blockIdx.y, slot = blockIdx.z / S, seg = blockIdx.z % S, tid = threadIdx.x;
    const int g = spill_g[slot], n_old = spill_n_old[slot];
    const int seg_lo = seg * seg_len, seg_hi = min(seg_lo + seg_len, M);
    const int k0 = max(n_old, seg_lo), k1 = min(n_old + g, seg_hi);   // new keys of this segment
    const size_t row = ((size_t)slot * Hkv + gi) * L + l;
    int32_t *off = offsets + (row * S + seg) * (size_t)(NB + 1);
    if (k0 >= k1) {
        // a segment beyond all keys gets the offsets a build writes there (every bucket empty at seg_lo), so that tables that
        // were never built end up identical to a rebuild too
        if (g > 0 && seg_lo >= n_old + g)
            for (int c = tid; c <= NB; c += T) off[c] = seg_lo;
        return;
    }
    uint16_t *it = items + row * (size_t)M + seg_lo;
    const int16_t *cn = codes + (size_t)spill_pre[slot] * Hkv * L + ((size_t)gi * L + l) * g - n_old;   // cn[key]
    const int base0 = off[0];
    const int32_t *oo = off;
    if (staged) {
        for (int c = tid; c <= NB; c += T) oo_s[c] = off[c];
        oo = oo_s;
    }
    for (int c = tid; c <= NB; c += T) ex[c] = 0;
    __syncthreads();
    for (int k = k0 + tid; k < k1; k += T) {
        const int c = cn[k];
        if (c >= 0 && c < NB) atomicAdd(&ex[c], 1);
    }
    __syncthreads();
    {   // exclusive scan of ex[0..NB) in place; ex[NB] = number of new keys
        const int per = (NB + T - 1) / T;
        const int c0 = min(tid * per, NB), c1 = min(c0 + per, NB);
        int local = 0;
        for (int c = c0; c < c1; ++c) local += ex[c];
        int total;
        int run = block_exclusive_scan(local, wsum, &total);
        for (int c = c0; c < c1; ++c) {
            const int h = ex[c];
            ex[c] = run;
            run += h;
        }
        if (tid == 0) ex[NB] = total;
    }
    __syncthreads();
    // old items, top chunk first
    const int old_cnt = oo[NB] - base0;
    for (int top = old_cnt; top > 0; top -= T * UN) {
        const int lo = max(0, top - T * UN);
        uint16_t v[UN];
        int dst[UN];
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const int p = lo + u * T + tid;
            dst[u] = -1;
            if (p < top) {
                int a = 0, z = NB;   // last bucket whose start is <= p: the bucket holding p
                while (z - a > 1) {
                    const int mid = (a + z) >> 1;
                    if (oo[mid] - base0 <= p) a = mid; else z = mid;
                }
                const int sh = ex[a];
                if (sh) {
                    v[u] = it[p];
                    dst[u] = p + sh;
                }
            }
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < UN; ++u)
            if (dst[u] >= 0) it[dst[u]] = v[u];
        __syncthreads();
    }
    // new keys behind the old items of their bucket; ex[c] ends as the inclusive prefix
    for (int k = k0 + tid; k < k1; k += T) {
        const int c = cn[k];
        if (c >= 0 && c < NB) it[oo[c + 1] - base0 + atomicAdd(&ex[c], 1)] = (uint16_t)(k - seg_lo);
    }
    __syncthreads();
    // every thread reads and rewrites only its own entries of `off` (base0 was read before the first barrier)
    for (int c = tid; c <= NB; c += T) off[c] = seg_lo + (oo[c] - base0) + (c ? ex[c - 1] : 0);
}

// ---------------------------------------------------------------------------------------------
// Table truncate of a compaction (mpig_compact_context, store.cu), the mirror of table_merge_kernel: drop from every bucket of a
// context slot's tables the items of keys >= lo[c], in place.  One CTA per (table, kv-head, slot x key segment); segments
// holding no key of [lo[c], hi[c]) return at once, so lo[c] == hi[c] leaves a slot untouched.  No assumption is made on where
// the dropped items sit inside a bucket: the segment's items are partitioned stably, kept ones moving down in ascending chunks
// (a kept item at position p lands at or below p, so a write never reaches a position a later chunk still has to read, and the
// block scan between the reads and the writes of a chunk orders them inside it).  With kc[c] = kept items of bucket c:
//   new offset of bucket c = seg_lo + sum of kc over the buckets before c
// A segment at or past lo keeps nothing: every bucket ends empty at seg_lo, what a build writes there.
// grid (L, Hkv, C * S), 512 threads; dynamic smem = (NB + 1 + 40 [+ NB + 1 when staged]) ints.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512) table_truncate_kernel(int32_t *offsets, uint16_t *items, const int32_t *__restrict__ lo_,
                                                             const int32_t *__restrict__ hi_, int Hkv, int L, int NB, int M, int S,
                                                             int seg_len, int staged) {
    extern __shared__ int smem_i[];
    constexpr int T = 512, UN = 8;
    int *kc = smem_i;                // NB + 1: kept items per bucket -> exclusive prefix
    int *wsum = smem_i + NB + 1;     // 40
    int *oo_s = wsum + 40;           // NB + 1 old offsets (staged)
    const int l = blockIdx.x, gi = blockIdx.y, slot = blockIdx.z / S, seg = blockIdx.z % S, tid = threadIdx.x;
    const int lo = lo_[slot], hi = hi_[slot];
    const int seg_lo = seg * seg_len, seg_hi = min(seg_lo + seg_len, M);
    if (max(lo, seg_lo) >= min(hi, seg_hi)) return;
    const size_t row = ((size_t)slot * Hkv + gi) * L + l;
    int32_t *off = offsets + (row * S + seg) * (size_t)(NB + 1);
    uint16_t *it = items + row * (size_t)M + seg_lo;
    const int lim = lo - seg_lo;   // items (key - seg_lo) below lim are kept
    const int base0 = off[0];
    const int32_t *oo = off;
    if (staged) {
        for (int c = tid; c <= NB; c += T) oo_s[c] = off[c];
        oo = oo_s;
    }
    for (int c = tid; c <= NB; c += T) kc[c] = 0;
    __syncthreads();
    const int cnt = oo[NB] - base0;
    for (int p = tid; p < cnt; p += T) {
        if ((int)it[p] >= lim) continue;
        int a = 0, z = NB;   // last bucket whose start is <= p: the bucket holding p
        while (z - a > 1) {
            const int mid = (a + z) >> 1;
            if (oo[mid] - base0 <= p) a = mid; else z = mid;
        }
        atomicAdd(&kc[a], 1);
    }
    __syncthreads();
    {   // exclusive scan of kc[0..NB) in place; kc[NB] = kept items
        const int per = (NB + T - 1) / T;
        const int c0 = min(tid * per, NB), c1 = min(c0 + per, NB);
        int local = 0;
        for (int c = c0; c < c1; ++c) local += kc[c];
        int total;
        int run = block_exclusive_scan(local, wsum, &total);
        for (int c = c0; c < c1; ++c) {
            const int h = kc[c];
            kc[c] = run;
            run += h;
        }
        if (tid == 0) kc[NB] = total;
    }
    __syncthreads();
    // stable partition: thread t of a chunk owns positions p0 + t*UN .. + UN - 1
    int out = 0;
    for (int p0 = 0; p0 < cnt; p0 += T * UN) {
        uint16_t v[UN];
        int keep = 0;
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const int p = p0 + tid * UN + u;
            v[u] = p < cnt ? it[p] : (uint16_t)0xffffu;
            keep += (p < cnt && (int)v[u] < lim);
        }
        int total;
        int dst = out + block_exclusive_scan(keep, wsum, &total);   // its barriers order every read above before any write below
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const int p = p0 + tid * UN + u;
            if (p < cnt && (int)v[u] < lim) it[dst++] = v[u];
        }
        out += total;
    }
    __syncthreads();
    // every thread rewrites only its own entries of `off` (base0 and, unstaged, oo were read before the barriers above)
    for (int c = tid; c <= NB; c += T) off[c] = seg_lo + kc[c];
}

// ---------------------------------------------------------------------------------------------
// Stage 2: probe.  A CLUSTER of C CTAs per q-head; CTA c of the cluster owns the key range
// [c*Mc, (c+1)*Mc) and keeps one small tag per key of its range in shared memory.
//
// No atomics.  Shared-memory atomics retire ~1 lane per 2 cycles on this part, which made the first
// (bitmap + atomicOr) version of this kernel the slowest of the three; the state machine of
// lsh.cc:272-283 is instead realised with two sweeps of PLAIN, idempotent stores:
//   sweep 1: every candidate (table t, key i) stores  tag[i] = t          (any one writer wins)
//   sweep 2: every candidate re-reads tag[i]; if it is not its own t, a second table also holds key i,
//            so it stores tag[i] = SEL.  A key hit by exactly one table keeps that table's id.
// Afterwards tag == EMPTY <=> 0 collisions, tag == table id <=> exactly 1, tag == SEL <=> >= 2, i.e. the
// reference's saturating mask byte {0,1,2}.  Every CTA of the cluster streams all L probed buckets
// (coalesced 128-byte chunks, one binary search per 32-candidate chunk, 4 chunks in flight per warp) and
// keeps only the candidates of its own key range; the per-range counts are exchanged through distributed
// shared memory (st.shared::cluster + cluster barrier) so that the cluster emits one ascending index list.
// dynamic smem: tag[Mc] | s_start[L] | s_len[L] | s_cpre[L+1] | s_counts[8] | wsum[40] | s_ctab[2048] u16
// ---------------------------------------------------------------------------------------------
template <typename TagT, int THREADS>
__global__ void __launch_bounds__(THREADS) probe_kernel(const int32_t *__restrict__ query,    // (H, L)
                                                        const int32_t *__restrict__ offsets,  // [BG][L][S][NB+1]
                                                        const uint16_t *__restrict__ items,   // [BG][L][M]
                                                        int32_t *__restrict__ results,        // (H, M)
                                                        int32_t *__restrict__ nnz,            // (H)
                                                        uint32_t *__restrict__ bitmaps_out,   // (H,2,words) or null
                                                        const int32_t *__restrict__ slot_of,  // (B) or null: request b reads slot b
                                                        const uint32_t *__restrict__ vis,     // [C][M] shared spill mode, else null
                                                        const int32_t *__restrict__ plo,      // [C] this layer's private starts
                                                        int L, int NB, int M, int G, int Hq, int Mc, int words, int S, int r, int seg_len) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    constexpr TagT SEL = (TagT)(~(TagT)0);
    constexpr TagT EMPTY = (TagT)(SEL - 1);
    constexpr int NWARPS = THREADS / 32;
    constexpr int UN = 4;
    TagT *tag = reinterpret_cast<TagT *>(smem_raw);
    int *s_start = reinterpret_cast<int *>(smem_raw + (((size_t)Mc * sizeof(TagT) + 15) & ~(size_t)15));
    int *s_len = s_start + L;
    int *s_cpre = s_len + L;
    int *s_counts = s_cpre + L + 1;
    int *wsum = s_counts + 16;
    uint16_t *s_ctab = reinterpret_cast<uint16_t *>(wsum + 40);
    constexpr int MAXCH = 2048;
    const unsigned C = cluster_nctarank(), c = cluster_ctarank();
    const int h = blockIdx.x / C, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // slot group of the head's tables.  The map may be read before griddepcontrol.wait: only copy-engine calls write it, and a
    // kernel starts after every copy ordered before it in the stream has completed (PDL overlaps a kernel with a kernel only)
    const int g = slot_of ? slot_of[h / Hq] * (Hq / G) + (h % Hq) / G : h / G;
    // CTA c of the cluster owns keys [lo_key, lo_key + Mc): sub-range (c % r) of key segment (c / r)
    const int seg = (int)c / r;
    const int lo_rel = ((int)c % r) * Mc;
    const int lo_key = seg * seg_len + lo_rel;
    const bool seg_ok = seg < S;

    cluster_arrive_relaxed();   // paired with the wait before the first distributed-shared-memory store
    {
        const uint32_t fillw = (sizeof(TagT) == 1) ? 0xFEFEFEFEu : 0xFFFEFFFEu;
        uint32_t *tw = reinterpret_cast<uint32_t *>(tag);
        for (int w = tid; w < (int)(Mc * sizeof(TagT) / 4); w += THREADS) tw[w] = fillw;
    }
    pdl_launch_dependents();  // let the attention kernel set up its barriers; it waits for this grid's results
    pdl_wait();               // query codes come from the SimHash kernel

    // bucket bounds of the L probed buckets (lsh.cc:266-271): two adjacent CSR entries each
    int my_chunks[(1024 + THREADS - 1) / THREADS];
#pragma unroll
    for (int r = 0; r < (1024 + THREADS - 1) / THREADS; ++r) {
        const int t = tid + r * THREADS;
        my_chunks[r] = 0;
        if (t < L) {
            const int code = query[(size_t)h * L + t];
            int s = 0, e = 0;
            if (seg_ok && code >= 0 && code < NB) {
                const int32_t *o = offsets + (((size_t)g * L + t) * S + seg) * (size_t)(NB + 1) + code;
                s = __ldg(o);
                e = __ldg(o + 1);
            }
            const int len = max(e - s, 0);
            s_start[t] = s;
            s_len[t] = len;
            my_chunks[r] = (len + 31) >> 5;
        }
    }
    int total_chunks = 0;
#pragma unroll
    for (int r = 0; r < (1024 + THREADS - 1) / THREADS; ++r) {
        if (r * THREADS < L) {  // uniform across the CTA
            int tot_r;
            const int ex = block_exclusive_scan(my_chunks[r], wsum, &tot_r);
            const int t = tid + r * THREADS;
            if (t < L) s_cpre[t] = total_chunks + ex;
            total_chunks += tot_r;
        }
    }
    if (tid == 0) s_cpre[L] = total_chunks;
    __syncthreads();

    // chunk -> table map (one entry per 32-candidate chunk), so that no search is needed per chunk
    for (int t = tid; t < L; t += THREADS) {
        const int c0 = s_cpre[t], c1 = min(s_cpre[t + 1], MAXCH);
        for (int ch = c0; ch < c1; ++ch) s_ctab[ch] = (uint16_t)t;
    }
    __syncthreads();

    const uint16_t *items_g = items + (size_t)g * L * (size_t)M;
    // the first KEEP chunks of every warp stay in registers between the two sweeps; every load of sweep 1 is
    // issued before the first tag is written, so the whole bucket stream costs one memory latency
    constexpr int KEEP = 16;
    int idx[KEEP];
    uint32_t tt_pack[KEEP / 2];  // two 16-bit table ids per register
    auto chunk_table = [&](int ch) -> int {
        if (ch < MAXCH) return (int)s_ctab[ch];
        int lo = 0, hi = L;  // beyond the map (pathologically long buckets): search
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (s_cpre[mid] <= ch) lo = mid; else hi = mid;
        }
        return lo;
    };
#pragma unroll
    for (int k = 0; k < KEEP; ++k) {
        const int ch = warp + k * NWARPS;
        idx[k] = -1;
        int t = 0;
        if (ch < total_chunks) {
            t = chunk_table(ch);
            const int e = ((ch - s_cpre[t]) << 5) + lane;
            if (e < s_len[t]) idx[k] = (int)__ldg(items_g + (size_t)t * M + s_start[t] + e);   // key - segment base
        }
        if (k & 1) tt_pack[k >> 1] |= (uint32_t)t << 16; else tt_pack[k >> 1] = (uint32_t)t;
    }
#pragma unroll
    for (int k = 0; k < KEEP; ++k) {
        const int i = idx[k] - lo_rel;
        idx[k] = (idx[k] >= 0 && i >= 0 && i < Mc) ? i : -1;  // keep only this CTA's key range
        if (idx[k] >= 0) tag[idx[k]] = (TagT)((tt_pack[k >> 1] >> ((k & 1) * 16)) & 0xffffu);   // 0 -> 1 (lsh.cc:276-277)
    }
    for (int ch = warp + KEEP * NWARPS; ch < total_chunks; ch += NWARPS) {  // overflow chunks (rare)
        const int t = chunk_table(ch);
        const int e = ((ch - s_cpre[t]) << 5) + lane;
        if (e < s_len[t]) {
            const int i = (int)__ldg(items_g + (size_t)t * M + s_start[t] + e) - lo_rel;
            if (i >= 0 && i < Mc) tag[i] = (TagT)t;
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < KEEP; ++k) {
        if (idx[k] >= 0 && tag[idx[k]] != (TagT)((tt_pack[k >> 1] >> ((k & 1) * 16)) & 0xffffu)) tag[idx[k]] = SEL;  // 1 -> 2
    }
    for (int ch = warp + KEEP * NWARPS; ch < total_chunks; ch += NWARPS) {
        const int t = chunk_table(ch);
        const int e = ((ch - s_cpre[t]) << 5) + lane;
        if (e < s_len[t]) {
            const int i = (int)__ldg(items_g + (size_t)t * M + s_start[t] + e) - lo_rel;
            if (i >= 0 && i < Mc && tag[i] != (TagT)t) tag[i] = SEL;
        }
    }
    __syncthreads();
    if (vis) {   // shared spill mode: the private keys of the slot that this head's request does not see (after pdl_wait above)
        const int sl = slot_of[h / Hq];
        filter_private(tag, vis + (size_t)sl * M, plo[sl], lo_key, Mc, h / Hq);
    }

    // compaction of this CTA's key range, ascending.  Each thread owns a run of `pw` 32-bit words of tags; pw is odd so the
    // lanes of a warp start in 32 different banks (an even word stride made every sweep load a 2..8-way bank conflict).
    constexpr int TPW = 4 / (int)sizeof(TagT);   // tags per word
    const int nwords = Mc / TPW;                 // Mc is a multiple of 32
    const int pw = ((nwords + THREADS - 1) / THREADS) | 1;
    const int w0 = min(tid * pw, nwords), w1 = min(w0 + pw, nwords);
    const uint32_t *tagw = reinterpret_cast<const uint32_t *>(tag);
    auto sel_count = [](uint32_t x) -> int {
        return (sizeof(TagT) == 1) ? (__popc(__vcmpeq4(x, 0xFFFFFFFFu)) >> 3) : (__popc(__vcmpeq2(x, 0xFFFFFFFFu)) >> 4);
    };
    int cnt = 0;
    for (int w = w0; w < w1; ++w) cnt += sel_count(tagw[w]);
    int tot;
    int pos = block_exclusive_scan(cnt, wsum, &tot);
    cluster_wait();   // every CTA of the cluster has started: remote stores are legal from here on
    if (tid == 0)
        for (unsigned rr = 0; rr < C; ++rr) st_shared_cluster_u32(&s_counts[c], rr, (uint32_t)tot);
    cluster_barrier();
    int base = 0, total_all = 0;
    for (unsigned rr = 0; rr < C; ++rr) {
        const int v = s_counts[rr];
        if (rr < c) base += v;
        total_all += v;
    }
    int32_t *res = results + (size_t)h * M + base;
    for (int w = w0; w < w1; ++w) {
        const uint32_t x = tagw[w];
        if (sel_count(x) == 0) continue;
#pragma unroll
        for (int b = 0; b < TPW; ++b)
            if ((TagT)(x >> (8 * (int)sizeof(TagT) * b)) == SEL) res[pos++] = lo_key + w * TPW + b;
    }
    if (c == 0 && tid == 0) nnz[h] = total_all;
    if (bitmaps_out) {
        uint32_t *bo = bitmaps_out + (size_t)h * 2 * words;
        for (int w = tid; w < Mc / 32; w += THREADS) {
            const int gw = lo_key / 32 + w;
            if (gw >= words || lo_rel + w * 32 >= seg_len) break;   // ranges are padded to 32 keys: stay inside this CTA's segment
            uint32_t b1 = 0, b2 = 0;
            for (int b = 0; b < 32; ++b) {
                const TagT v = tag[w * 32 + b];
                b1 |= (uint32_t)(v != EMPTY) << b;
                b2 |= (uint32_t)(v == SEL) << b;
            }
            bo[gw] = b1;
            bo[words + gw] = b2;
        }
    }
}

// LSH::get_mask: bytes {0,1,2} from the two saved bitmaps
__global__ void expand_mask_kernel(const uint32_t *__restrict__ bitmaps, uint8_t *__restrict__ mask, int M, int words) {
    const int h = blockIdx.y;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= M) return;
    const uint32_t *b = bitmaps + (size_t)h * 2 * words;
    const uint32_t bit = 1u << (j & 31);
    mask[(size_t)h * M + j] = (uint8_t)(((b[j >> 5] & bit) ? 1 : 0) + ((b[words + (j >> 5)] & bit) ? 1 : 0));
}

// diagnostic: full collision counts (library/lsh/test.py:43)
__global__ void collision_counts_kernel(const int32_t *__restrict__ query, const int32_t *__restrict__ offsets,
                                        const uint16_t *__restrict__ items, int32_t *__restrict__ counts,
                                        const int32_t *__restrict__ slot_of, int L, int NB, int M, int G, int Hq, int S, int seg_len) {
    const int h = blockIdx.x, g = slot_of ? slot_of[h / Hq] * (Hq / G) + (h % Hq) / G : h / G;
    for (int t = 0; t < L; ++t) {
        const int code = query[(size_t)h * L + t];
        if (code < 0 || code >= NB) continue;
        const uint16_t *it = items + ((size_t)g * L + t) * (size_t)M;
        for (int sg = 0; sg < S; ++sg) {
            const int32_t *o = offsets + (((size_t)g * L + t) * S + sg) * (size_t)(NB + 1) + code;
            const int s = o[0], e = o[1];
            for (int j = s + threadIdx.x; j < e; j += blockDim.x) {
                const int i = sg * seg_len + (int)it[j];
                if (i < M) atomicAdd(&counts[(size_t)h * M + i], 1);
            }
        }
    }
}

}  // namespace mpig

using namespace mpig;

namespace mpig {
// shared with decode.cu
template <typename TagT, int T>
static int launch_probe_tt(mpig_ctx *ctx, int layer, const int32_t *query, int32_t *results, int32_t *nnz,
                           cudaStream_t s, bool pdl, int C, int r, int Mc, size_t smem) {
    const LayerStore &ls = ctx->layers[layer];
    const int M = ctx->cfg.max_length, L = ctx->cfg.L, S = ctx->nseg;
    MPIG_FUNC_ATTR((probe_kernel<TagT, T>), cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    MPIG_FUNC_ATTR((probe_kernel<TagT, T>), cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    uint32_t *bm = ctx->save_mask ? ctx->bitmaps : nullptr;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(ctx->H * C);
    cfg.blockDim = dim3(T);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 2 : 1;
    MPIG_CUDA(cudaLaunchKernelEx(&cfg, probe_kernel<TagT, T>, query, (const int32_t *)ls.offsets, (const uint16_t *)ls.items,
                                 results, nnz, bm, ctx->slot_map(), ctx->vis_map(), ctx->private_lo_map(layer), L,
                                 ctx->NB, M, ctx->G, ctx->cfg.num_attention_heads, Mc,
                                 ctx->bitmap_words, S, r, ctx->seg_len));
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

// Cluster geometry of a probe (shared with the fused decode kernel): S key segments (padded to a power of two Sp; CTAs of the
// padding segments have nothing to scan) x r CTAs per segment (r a power of two), spreading each head over as many SMs as the
// grid leaves free; the tag array of one CTA covers at most one segment (<= 65536 keys) so it always fits in shared memory.
ProbeGeom probe_geometry(const mpig_ctx *ctx) {
    ProbeGeom gm;
    gm.Sp = 1;
    while (gm.Sp < ctx->nseg) gm.Sp *= 2;
    gm.r = 1;
    while (gm.Sp * gm.r * 2 <= ctx->max_cluster && ctx->H * gm.Sp * gm.r * 2 <= ctx->cta_per_sm * ctx->num_sms) gm.r *= 2;
    gm.C = gm.Sp * gm.r;
    gm.Mc = ((ctx->seg_len + gm.r - 1) / gm.r + 31) & ~31;
    return gm;
}

template <typename TagT>
static int launch_probe_t(mpig_ctx *ctx, int layer, const int32_t *query, int32_t *results, int32_t *nnz,
                          cudaStream_t s, bool pdl) {
    const int M = ctx->cfg.max_length, L = ctx->cfg.L;
    const ProbeGeom gm = probe_geometry(ctx);
    MPIG_REQUIRE(gm.Sp <= 16, MPIG_EUNSUPPORTED, "probe: max_length=%d needs %d key segments (> 16)", M, ctx->nseg);
    const int C = gm.C, r = gm.r, Mc = gm.Mc;
    const size_t smem = (((size_t)Mc * sizeof(TagT) + 15) & ~(size_t)15) + (size_t)(3 * L + 1 + 16 + 40) * sizeof(int) + 2048 * 2 + 16;
    MPIG_REQUIRE(smem <= 220 * 1024, MPIG_EUNSUPPORTED, "probe: L=%d needs %zu B of shared memory per CTA", L, smem);
    // more clusters than the GPU holds at once (1024-thread CTAs are one per SM): halve the CTA so two share an SM and the
    // whole grid is resident in one wave
    if (ctx->H * C > ctx->num_sms && smem <= 110 * 1024)
        return launch_probe_tt<TagT, 512>(ctx, layer, query, results, nnz, s, pdl, C, r, Mc, smem);
    return launch_probe_tt<TagT, 1024>(ctx, layer, query, results, nnz, s, pdl, C, r, Mc, smem);
}

int launch_probe(mpig_ctx *ctx, int layer, const int32_t *query, int32_t *results, int32_t *nnz, cudaStream_t s, bool pdl) {
    // table ids 0..L-1 must stay clear of the two reserved tag values
    if (ctx->cfg.L <= 254) return launch_probe_t<uint8_t>(ctx, layer, query, results, nnz, s, pdl);
    return launch_probe_t<uint16_t>(ctx, layer, query, results, nnz, s, pdl);
}
}  // namespace mpig

// one launch builds every (kv-head, table, segment) of a request; idx == nullptr: codes are per key (device route),
// else codes/idx are the sorted codes and their argsort (LSH::fill route)
static int launch_build(mpig_ctx *ctx, int layer, int request, const int16_t *codes, const int32_t *idx, int n, cudaStream_t s) {
    const LayerStore &ls = ctx->layers[layer];
    const int Hkv = ctx->cfg.num_key_value_heads, L = ctx->cfg.L, S = ctx->nseg, M = ctx->cfg.max_length;
    const size_t slot = ctx->h_slot_of[request];   // every request bound to this slot sees the new tables
    int32_t *off = ls.offsets + slot * Hkv * L * S * (size_t)(ctx->NB + 1);
    uint16_t *it = reinterpret_cast<uint16_t *>(ls.items) + slot * Hkv * L * (size_t)M;
    const size_t base = (size_t)(ctx->NB + 1 + 40) * sizeof(int);
    const int staged = base + (size_t)ctx->seg_len * 2 <= 200 * 1024;   // stage the sorted segment in shared memory when it fits
    const size_t smem = base + (staged ? (size_t)ctx->seg_len * 2 : 0);
    MPIG_FUNC_ATTR(build_segments_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    MPIG_FUNC_ATTR(build_segments_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (idx)
        build_segments_kernel<true><<<dim3(L, Hkv, S), 1024, smem, s>>>(codes, idx, off, it, n, ctx->NB, M, L, S, staged, ctx->seg_len);
    else
        build_segments_kernel<false><<<dim3(L, Hkv, S), 1024, smem, s>>>(codes, nullptr, off, it, n, ctx->NB, M, L, S, staged, ctx->seg_len);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

int mpig::launch_table_merge(mpig_ctx *ctx, int layer, const int16_t *codes, const int32_t *g, const int32_t *pre,
                             const int32_t *n_old, cudaStream_t s) {
    const LayerStore &ls = ctx->layers[layer];
    const int Hkv = ctx->cfg.num_key_value_heads, L = ctx->cfg.L, S = ctx->nseg, NB = ctx->NB;
    const size_t base = (size_t)(NB + 1 + 40) * sizeof(int);
    const int staged = base + (size_t)(NB + 1) * sizeof(int) <= 200 * 1024;   // K <= 14
    const size_t smem = base + (staged ? (size_t)(NB + 1) * sizeof(int) : 0);
    MPIG_FUNC_ATTR(table_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    table_merge_kernel<<<dim3(L, Hkv, ctx->C * S), 512, smem, s>>>(codes, ls.offsets, reinterpret_cast<uint16_t *>(ls.items), g, pre,
                                                                   n_old, Hkv, L, NB, ctx->cfg.max_length, S, ctx->seg_len, staged);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

int mpig::launch_table_truncate(mpig_ctx *ctx, int layer, const int32_t *lo, const int32_t *hi, cudaStream_t s) {
    const LayerStore &ls = ctx->layers[layer];
    const int Hkv = ctx->cfg.num_key_value_heads, L = ctx->cfg.L, S = ctx->nseg, NB = ctx->NB;
    const size_t base = (size_t)(NB + 1 + 40) * sizeof(int);
    const int staged = base + (size_t)(NB + 1) * sizeof(int) <= 200 * 1024;   // K <= 14
    const size_t smem = base + (staged ? (size_t)(NB + 1) * sizeof(int) : 0);
    MPIG_FUNC_ATTR(table_truncate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    table_truncate_kernel<<<dim3(L, Hkv, ctx->C * S), 512, smem, s>>>(ls.offsets, reinterpret_cast<uint16_t *>(ls.items), lo, hi, Hkv,
                                                                      L, NB, ctx->cfg.max_length, S, ctx->seg_len, staged);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

extern "C" {

int mpig_lsh_fill(mpig_ctx *ctx, int layer, int request, const int16_t *sorted_codes, const int32_t *sorted_indices,
                  int n, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_lsh_fill");
    if (rc) return rc;
    MPIG_REQUIRE(request >= 0 && request < ctx->cfg.batch_size, MPIG_EINVAL, "mpig_lsh_fill: request %d out of range", request);
    MPIG_REQUIRE(n >= 0 && n <= ctx->cfg.max_length, MPIG_EINVAL, "mpig_lsh_fill: n=%d exceeds max_length=%d", n,
                 ctx->cfg.max_length);
    MPIG_REQUIRE(n == 0 || (sorted_codes && sorted_indices), MPIG_EINVAL, "mpig_lsh_fill: null input");
    rc = refresh_maps(ctx, as_stream(stream));   // the tables of the slot the request is bound to now
    if (rc) return rc;
    rc = reset_private(ctx, layer, request, n, as_stream(stream));
    if (rc) return rc;
    return launch_build(ctx, layer, request, sorted_codes, sorted_indices, n, as_stream(stream));
}

int mpig_lsh_build(mpig_ctx *ctx, int layer, int request, const int16_t *key_codes, int n, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_lsh_build");
    if (rc) return rc;
    MPIG_REQUIRE(request >= 0 && request < ctx->cfg.batch_size, MPIG_EINVAL, "mpig_lsh_build: request %d out of range", request);
    MPIG_REQUIRE(n >= 0 && n <= ctx->cfg.max_length, MPIG_EINVAL, "mpig_lsh_build: n=%d exceeds max_length=%d", n,
                 ctx->cfg.max_length);
    MPIG_REQUIRE(n == 0 || key_codes, MPIG_EINVAL, "mpig_lsh_build: null input");
    rc = refresh_maps(ctx, as_stream(stream));   // the tables of the slot the request is bound to now
    if (rc) return rc;
    rc = reset_private(ctx, layer, request, n, as_stream(stream));
    if (rc) return rc;
    return launch_build(ctx, layer, request, key_codes, nullptr, n, as_stream(stream));
}

int mpig_lsh_batch_retrieve(mpig_ctx *ctx, int layer, const int32_t *query, int32_t *results, int32_t *nnz, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_lsh_batch_retrieve");
    if (rc) return rc;
    MPIG_REQUIRE(query && results && nnz, MPIG_EINVAL, "mpig_lsh_batch_retrieve: null argument");
    return launch_probe(ctx, layer, query, results, nnz, as_stream(stream), false);
}

int mpig_lsh_get_mask(mpig_ctx *ctx, uint8_t *mask_out, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx && mask_out, MPIG_EINVAL, "mpig_lsh_get_mask: null argument");
    MPIG_REQUIRE(ctx->save_mask, MPIG_ESTATE,
                 "mpig_lsh_get_mask: enable mpig_set_option(ctx, \"save_mask\", 1) before the probe");
    const int M = ctx->cfg.max_length;
    expand_mask_kernel<<<dim3((M + 255) / 256, ctx->H), 256, 0, as_stream(stream)>>>(ctx->bitmaps, mask_out, M,
                                                                                    ctx->bitmap_words);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

int mpig_lsh_collision_counts(mpig_ctx *ctx, int layer, const int32_t *query, int32_t *counts, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_lsh_collision_counts");
    if (rc) return rc;
    MPIG_REQUIRE(query && counts, MPIG_EINVAL, "mpig_lsh_collision_counts: null argument");
    const LayerStore &ls = ctx->layers[layer];
    MPIG_CUDA(cudaMemsetAsync(counts, 0, (size_t)ctx->H * ctx->cfg.max_length * sizeof(int32_t), as_stream(stream)));
    collision_counts_kernel<<<ctx->H, 256, 0, as_stream(stream)>>>(query, ls.offsets, reinterpret_cast<const uint16_t *>(ls.items), counts,
                                                                  ctx->slot_map(), ctx->cfg.L, ctx->NB, ctx->cfg.max_length, ctx->G,
                                                                  ctx->cfg.num_attention_heads, ctx->nseg, ctx->seg_len);
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

int mpig_lsh_table_ptrs(mpig_ctx *ctx, int layer, const int32_t **offsets, const uint16_t **items) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    int rc = check_layer(ctx, layer, true, "mpig_lsh_table_ptrs");
    if (rc) return rc;
    if (offsets) *offsets = ctx->layers[layer].offsets;
    if (items) *items = reinterpret_cast<const uint16_t *>(ctx->layers[layer].items);
    return MPIG_OK;
}

}  // extern "C"
