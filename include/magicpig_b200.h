/*
 * magicpig_b200.h -- C ABI of the H100-native (sm_90a) LSH-sampled sparse-attention decode path.
 *
 * This is the drop-in boundary for ONE hot path of Infini-AI-Lab/MagicPIG: everything that
 * `models/attnserver.py::LSHSparseAttnServer.decode` (attnserver.py:228-312) does for a sparse
 * layer -- SimHash of the decode queries, the probe of the L hash tables, the importance-weighted
 * gather attention and the LSE merge with the sink/local/generated window -- with the KV cache and
 * the hash tables resident in HBM.  The entry points below are what the reference's two pybind
 * modules bind for this path:
 *
 *     lsh.LSH                              (library/lsh/lsh.cc:316-326,  class lsh.h:14-43)
 *     sparse_attention_cpu.SparseAttentionServer
 *                                          (library/sparse_attention/sparse_attention.cc:1243-1263,
 *                                           class sparse_attention.h:14-52)
 *
 * plus the GPU-side torch/FlashInfer glue of attnserver.py:264-310 that becomes kernels here.
 * Each function cites the reference interface it replaces.  INTEGRATION.md shows the binding a
 * MagicPIG maintainer would add.
 *
 * Conventions
 *   - plain C, opaque context, no torch types.  All tensor arguments are raw pointers to
 *     contiguous row-major arrays; `bf16` data is passed as `const void*` / `uint16_t` bits.
 *   - unless a function name ends in `_host`, pointers are DEVICE pointers on the context's
 *     device and work is enqueued on `stream` (a `cudaStream_t` passed as void*; NULL = legacy
 *     default stream).  Nothing synchronises the host; every call is CUDA-graph capturable.
 *     `*_host` entry points take HOST pointers (pinned for full speed), copy in/out on `stream`
 *     and return after the stream has drained -- the same synchronous host-buffer contract the
 *     reference's CPU operators have (attnserver.py:272-273, 299-303).
 *   - every function returns MPIG_OK (0) or a negative MPIG_E* code; mpig_last_error() gives the
 *     text.  Unlike the reference (asserts compiled out by -DNDEBUG -> silent UB) shape errors
 *     are reported.
 *   - indices: B batch (requests), Hq q-heads, Hkv kv-heads, G = Hq/Hkv, d head_dim (128),
 *     M = max_length, n = number of offloaded keys of a request, NB = 2^K buckets per table,
 *     "head" = b*Hq + h in [0, B*Hq), "group" = head / G in [0, B*Hkv)  (lsh.cc:251).
 *
 * There is NO CPU fallback anywhere behind this interface.
 */
#ifndef MAGICPIG_B200_H
#define MAGICPIG_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPIG_ABI_VERSION 1

enum {
    MPIG_OK = 0,
    MPIG_EINVAL = -1,   /* bad argument / shape */
    MPIG_ECUDA = -2,    /* CUDA runtime error (text in mpig_last_error) */
    MPIG_ENOMEM = -3,   /* device allocation failed */
    MPIG_ESTATE = -4,   /* call sequence error (e.g. layer not allocated, dense layer) */
    MPIG_EUNSUPPORTED = -5
};

typedef struct mpig_ctx mpig_ctx;

/* Mirrors the constructor arguments of LSHSparseAttnServer (attnserver.py:9-20) and of
 * LSH::alloc (lsh.cc:44-51) / SparseAttentionServer::alloc (sparse_attention.cc:546-552). */
typedef struct mpig_config {
    int32_t abi_version;          /* = MPIG_ABI_VERSION */
    int32_t device;               /* CUDA device ordinal */
    int32_t K;                    /* bits per table, 1..15 (int16 key codes, attnserver.py:69) */
    int32_t L;                    /* tables */
    int32_t num_layers;
    int32_t num_attention_heads;  /* Hq  (per rank under KV-head tensor parallelism) */
    int32_t num_key_value_heads;  /* Hkv (per rank) */
    int32_t head_dim;             /* d; 128 supported */
    int32_t batch_size;           /* B */
    int32_t max_length;           /* M: row capacity per (request, kv-head) */
    int32_t num_sink_tokens;      /* attnserver.py:13 (4) */
    int32_t num_local_tokens;     /* attnserver.py:14 (64) */
    int32_t generation_buffer;    /* attnserver.py:15 (256); window capacity = sink+local+generation_buffer */
    int32_t num_dense_layers;     /* entries used in dense_layers[] */
    int32_t dense_layers[16];     /* attnserver.py:18; tables/offload store are NOT allocated for these */
    int32_t alloc_dense_kv;       /* 1: also own the dense layers' full KV cache + dense decode kernel */
    int32_t ctas_per_sm;          /* probing / fused clusters planned for: 0 or 1 = one 1024-thread CTA per SM, 2 = two 512-thread
                                   * CTAs per SM (experiment switch); anything else is MPIG_EINVAL */
    /* number of context slots C in [0, batch_size]; 0 means C = batch_size (every request owns its slot).  The sampled store
     * and the L hash tables of every sparse layer exist once per SLOT; the window, avg_k, the dense layers' KV, the lengths and
     * the per-step scratch stay per REQUEST.  Request b is bound to slot b mod C at creation and after mpig_clear;
     * mpig_fork_request / mpig_bind_request change the binding.  Requests bound to one slot decode over one copy of the context
     * (parallel sampling, several questions about one document). */
    int32_t num_contexts;
    /* dense tail rows R; 0 (default) = every request owns a full dense KV cache [Hkv][max_length].  R > 0 (only with
     * 0 < C < batch_size, alloc_dense_kv = 1 and R <= max_length; otherwise MPIG_EINVAL) shares the dense layers' prompt too:
     * per dense layer a slot store [C][Hkv][max_length] and a tail [B][Hkv][R] per request.  mpig_dense_fill writes the rows of
     * the slot the request is bound to and makes seq_len the request's base; mpig_fork_request copies only src's rows past its
     * base; a request's dense capacity is min(max_length, base + R) (the plans refuse past it, a captured plan saturates and
     * raises mpig_error_flags bit 1); a rebound request must be dense-filled before its dense outputs mean anything;
     * dense_impl = 0 is MPIG_EUNSUPPORTED.  mpig_get_info("dense_tail_rows") reports R. */
    int32_t dense_tail_rows;
    /* 1 = shared spill (only with 0 < C < batch_size <= 32; otherwise MPIG_EINVAL).  mpig_spill_window accepts requests that
     * share a slot: their rows go into the slot's store and tables in request order, and every spilled key is PRIVATE:
     * request b samples the slot's prompt keys plus the private keys it spilled itself or inherited through mpig_fork_request,
     * so its result equals that of an exclusive slot holding those keys (codes, nnz and index sets equal after renumbering,
     * fp32 outputs up to summation order).  The capacity is shared (prompt + all private keys of a slot <= max_length).  A fill
     * of a slot (mpig_attn_fill, mpig_lsh_build / mpig_lsh_fill) and mpig_clear drop its private keys; private keys nobody
     * sees any more keep their rows until then, or until mpig_compact_context reclaims them.  mpig_lsh_collision_counts stays
     * unfiltered.  mpig_get_info("shared_spill") reports the flag. */
    int32_t shared_spill;
    int32_t reserved[4];          /* must be zero (MPIG_EINVAL otherwise) */
} mpig_config;

/* ---- lifetime ------------------------------------------------------------------------------- */
int mpig_create(const mpig_config *cfg, mpig_ctx **out);
void mpig_destroy(mpig_ctx *ctx);
const char *mpig_last_error(void);
int mpig_abi_version(void);
/* bytes of HBM owned by the context */
size_t mpig_device_bytes(const mpig_ctx *ctx);

/* Runtime knobs (no reference equivalent; the reference's are compile-time #defines such as
 * LSH_THREADS lsh.h:12 / ATTENTION_THREADS sparse_attention.h:10).  Unknown keys return MPIG_EINVAL.
 *   "save_mask"       0/1: keep the probe's collision bitmaps for mpig_lsh_get_mask (and, in the fused decode, write the
 *                     ascending index list and the query codes to HBM for mpig_last_probe; off = only nnz leaves the SMs)
 *   "decode_impl"     1 = ONE fused launch per sparse layer (fused.cu; default, used wherever its shape rules hold: L <= 1012
 *                     -- one-byte tags, passes of 253 tables --; any batch: one CTA per head in several waves once B*Hq > 2 * #SMs), 0 = three launches SimHash | probe | attend
 *   "fused_selcap"    selected keys a CTA of the fused kernel lists per pass (default 2048; tests lower it to force passes)
 *   "fused_kreg"      0 = whole 512-byte records through TMA + ldmatrix (default); 1 = the K half of each sampled record goes
 *                     from HBM straight into the tensor-core operand registers (LSU loads) and only the V half is staged in
 *                     shared memory by the TMA engine (more rows in flight per SM, measured slower: the L1 miss path caps it)
 *   "fused_issue_win" warps of a fused-kernel CTA that issue their tile's row requests at the same time, in warp order (default 8;
 *                     0 = all at once; 0..32).  Results do not depend on it; measured optimum 6..8 at every BASELINE shape
 *   "out_f32"         0/1: also keep the attention output BEFORE the ABI's bf16 rounding (fp32, read with mpig_last_out_f32);
 *                     this is where the parity tests apply the 1e-3 bar
 *   "attend_tma"      stand-alone gather kernel: 1 = per-row cp.async.bulk copies (default), 0 = per-row 16-B cp.async copies
 *   "attend_ctas" / "attend_warps"   grid / CTA shape of the stand-alone gather kernel (0 = automatic)
 *   "dense_impl"      1 = GQA-shared dense kernel (default), 0 = the gather kernel in range mode
 *   "keyhash_impl"    1 = persistent warp-specialised wgmma pipeline (default), 0 = one tile per CTA
 *   "pdl_first"       1 = launch the first kernel of mpig_decode with programmatic stream serialization too (default)
 *   "attend_skip" / "attend_debug" / "fused_debug" / "keyhash_skip"   timing-only elimination switches and clock stamps
 *                     (results are WRONG while a skip bit is set; used by scripts/kernel_bench.py and scripts/keyhash_bench.py) */
int mpig_set_option(mpig_ctx *ctx, const char *key, int64_t value);
/* Read-only facts: "last_decode_fused" (1 if the last mpig_decode ran the fused kernel), "fused_applicable",
 * "fused_cluster_waves" (waves of thread-block clusters one fused launch takes on this device; 1 = all resident at once,
 * 0 = fused decode not applicable), "window_capacity" (sink + local + generation_buffer rows), "table_segments" (key segments S
 * of the tables, see mpig_lsh_table_ptrs), "query_tokens_max" (t_max of mpig_reserve_query_tokens, 1 without), "tokens_cluster_waves"
 * (waves of clusters the last mpig_decode_tokens launch with T > 1 took), "num_contexts" (context slots C, see mpig_config), "dense_tail_rows" (R),
 * "shared_spill" (0 / 1), "chunk_tokens_max" (t_max of mpig_reserve_chunk_tokens, 0 without), "chunk_splits"
 * (key splits of the last mpig_chunk_attend launch, 0 before any). */
int mpig_get_info(mpig_ctx *ctx, const char *key, int64_t *value);
/* Capacity errors the DEVICE detected (the lengths saturate there): bit 0 = a sparse window is full (generation_buffer
 * exhausted: each further token overwrites the previous one's K/V), bit 1 = a dense cache reached its capacity (max_length, or base + R with dense_tail_rows = R), bit 2 = mpig_rewind
 * met a drop outside [0, T] (that request was left untouched), bit 3 = mpig_plan_tree met a malformed tree (that request ran as a
 * chain) or mpig_accept met a path that is not a root path of the step (that request was left untouched), bit 4 =
 * mpig_reorder_requests met a map that breaks its rule (every request was left untouched).  mpig_plan
 * itself returns MPIG_ESTATE for the same conditions as long as it has not been captured into a CUDA graph (replays advance
 * only the device-side lengths).  mpig_spill_window is the way out of a full sparse window.  Synchronises `stream`.  The
 * reference has no such check (flashinfer append past the page). */
int mpig_error_flags(mpig_ctx *ctx, int32_t *flags_out, void *stream);

/* LSHSparseAttnServer.clear (attnserver.py:314-331) = LSH::clear (lsh.cc:293-306) +
 * SparseAttentionServer::clear (sparse_attention.cc:586-598): forget all requests. */
int mpig_clear(mpig_ctx *ctx, void *stream);

/* hash_func: bf16 (d, K*L) row-major, column l*K+i = bit i of table l (attnserver.py:55,268-270). */
int mpig_set_hash_func(mpig_ctx *ctx, const void *hash_func_bf16, void *stream);

/* ---- context slots (no reference equivalent; see mpig_config.num_contexts) -------------------------------------------------
 * Fork and bind return MPIG_ESTATE when C = batch_size (the bindings are then fixed: request b reads slot b), are not capturable
 * (mpig_reorder_requests is the capturable form of a batch of forks), and
 * end the pending step: mpig_rewind / mpig_accept are refused (MPIG_ESTATE) until the next plan.  A step captured before either
 * call replays with the new bindings (the kernels read the device map).
 *
 * Bind `dst` to the slot of `src` and make dst's per-request state a copy of src's: for every sparse layer window rows
 * [0, win_len[src]) of every kv-head and avg_k, for every dense layer KV rows [0, dense_len[src]) of every kv-head, and both
 * lengths (device and host mirror).  Reads the device lengths and synchronises `stream` (correct after replays of a captured
 * plan); copy-engine calls only, plus in shared spill mode (shared_spill) one kernel: dst then sees exactly the private keys src
 * sees, and no longer its own.  MPIG_EINVAL: src == dst or either outside [0, batch_size). */
int mpig_fork_request(mpig_ctx *ctx, int src, int dst, void *stream);
/* Bind `request` to `slot` (in [0, C)); its window and lengths are left alone: fill the slot (mpig_attn_fill + mpig_lsh_build /
 * mpig_lsh_fill) and the window next.  In shared spill mode the request sees no private key until it spills again.  Synchronises
 * `stream`. */
int mpig_bind_request(mpig_ctx *ctx, int request, int slot, void *stream);
/* Request b continues request src_of[b]'s sequence (device int32 [B]; src_of[b] == b leaves b as it is).  The device-side,
 * capturable form of mpig_fork_request(src_of[b], b) for every b with src_of[b] != b, all at once (beam search: each step, each new
 * beam continues some old beam).  For every moved request b, with s = src_of[b]: window rows [0, win_len[s]) of every sparse layer
 * and kv-head and avg_k; dense rows [0, dense_len[s]) (dense_tail_rows = R > 0: tail rows [0, min(dense_len[s] - dense_base[s], R))
 * and the base); both lengths; the slot binding; in shared spill mode (shared_spill) b then sees exactly the private keys s sees.
 * Every later decode output equals the output after those forks, bitwise.  One kernel launch plus one device-to-device copy of
 * the slot map (the decode kernels read the map before they wait on their predecessor, so no kernel writes it).
 * The map's rule: 0 <= src_of[b] < B and src_of[src_of[b]] == src_of[b] for every b -- a request that is a source keeps its own
 * sequence, so no request is both read and written and the copy runs in place.  Any beam step can be put in this form
 * (magicpig_b200.attnserver.beam_sources).  A map that breaks the rule changes nothing and raises mpig_error_flags bit 4; outside
 * a capture the call reads the map first (synchronises `stream`) and then also returns MPIG_EINVAL (the call may be repeated).
 * Capturable: a replay applies whatever the map holds then.  Capturing it makes the host mirror of the lengths inexact until
 * mpig_clear (as a captured plan does), and makes every later host path that needs a request's binding or dense base (fills,
 * mpig_spill_window, fork, bind) read the device maps first, for the rest of the context's life (the graph may be replayed at
 * any time).  Eager calls leave the mirrors exact.  Ends the pending step (mpig_rewind / mpig_accept are refused until the next plan).  MPIG_ESTATE when
 * C = batch_size, MPIG_EINVAL on a null argument.  With R = 0 a moved request copies its whole dense cache: correct but slow at long
 * contexts (see DESIGN.md section 3.13). */
int mpig_reorder_requests(mpig_ctx *ctx, const int32_t *src_of, void *stream);

/* ---- lsh.LSH --------------------------------------------------------------------------------- */
/* LSH::fill (lsh.cc:143-201): tables of one (layer, request) from codes already sorted per
 * (kv-head, table).  sorted_codes int16 (Hkv, L, n); sorted_indices int32 (Hkv, L, n).  The tables are those of the slot `request`
 * is bound to (as for mpig_lsh_build and mpig_attn_fill): the fill changes the context of every request bound to that slot. */
int mpig_lsh_fill(mpig_ctx *ctx, int layer, int request, const int16_t *sorted_codes,
                  const int32_t *sorted_indices, int n, void *stream);
/* Key-side SimHash (attnserver.py:159-168): codes int16 (Hkv, L, n) of keys bf16 (Hkv, n, d) [already centred], with the
 * context's hash_func.  wgmma tensor-core GEMM whose epilogue keeps only the sign bits. */
int mpig_hash_keys(mpig_ctx *ctx, const void *keys_bf16, int n, int16_t *codes_out, void *stream);
/* Device-side replacement of `sort()` + LSH::fill (attnserver.py:186-193 + lsh.cc:143-201):
 * counting-sort the UNSORTED key codes int16 (Hkv, L, n) straight into the CSR tables. */
int mpig_lsh_build(mpig_ctx *ctx, int layer, int request, const int16_t *key_codes, int n, void *stream);
/* LSH::batch_retrieve (lsh.cc:210-241, retrieve :243-288).  query int32 (B*Hq, L);
 * results int32 (B*Hq, M): first nnz[head] entries valid, ASCENDING key index (the reference
 * emits second-hit order and pins only the set, library/lsh/test.py:47-56); nnz int32 (B*Hq). */
int mpig_lsh_batch_retrieve(mpig_ctx *ctx, int layer, const int32_t *query, int32_t *results,
                            int32_t *nnz, void *stream);
/* LSH::get_mask (lsh.cc:308-314): saturating collision counters {0,1,2} of the LAST probe,
 * uint8 (B*Hq, M), written to `mask_out`. */
int mpig_lsh_get_mask(mpig_ctx *ctx, uint8_t *mask_out, void *stream);
/* Full (unsaturated) collision counts of `query` against the tables of `layer`, int32 (B*Hq, M).
 * Diagnostic used by the parity tests (library/lsh/test.py:43 computes the same sum). */
int mpig_lsh_collision_counts(mpig_ctx *ctx, int layer, const int32_t *query, int32_t *counts, void *stream);
/* raw views for tests.  Segmented compact CSR: keys are cut into S = ceil(max_length / 65536) segments of equal length
 * seg_len = ceil(max_length / S) rounded up to 64; offsets int32 (C, Hkv, L, S, NB+1) = absolute bucket starts inside the item
 * row, items uint16 (C, Hkv, L, M) = key index - seg_len * segment, segment s occupying [s * seg_len, ...) of its row (C context
 * slots, the leading dimension). */
int mpig_lsh_table_ptrs(mpig_ctx *ctx, int layer, const int32_t **offsets, const uint16_t **items);

/* ---- sparse_attention_cpu.SparseAttentionServer ---------------------------------------------- */
/* SparseAttentionServer::fill (sparse_attention.cc:601-627).  k, v bf16 (Hkv, n, d);
 * kn fp32 (Hkv, n) = L2 norm of each (centred) key row as the caller computed it. */
int mpig_attn_fill(mpig_ctx *ctx, int layer, int request, const void *k_bf16, const void *v_bf16,
                   const float *kn, int n, void *stream);
/* SparseAttentionServer::attention_wrapper (sparse_attention.cc:629-745; math :38-240,:321-347).
 * K, L: the LSH parameters of the importance weights (the reference passes them per call too).
 * output bf16 (B*Hq, d); max_value_expsum fp32 (2, B*Hq): row 0 = m*log2(e), row 1 = base-2 LSE;
 * query bf16 (B*Hq, d); query_norm fp32 (B*Hq); ind int32 (B*Hq, M); nnz int32 (B*Hq). */
int mpig_attention_wrapper(mpig_ctx *ctx, int layer, int K, int L, void *output_bf16, float *max_value_expsum,
                           const void *query_bf16, const float *query_norm, const int32_t *ind,
                           const int32_t *nnz, void *stream);
/* get_key_cache / get_value_cache / get_key_norm (sparse_attention.cc:1213-1234), copied out
 * of the interleaved HBM layout: k, v bf16 (C, Hkv, M, d) and/or kn fp32 (C, Hkv, M), one entry per context slot (C = B unless
 * num_contexts says otherwise; request b's store is entry slot-of-b); NULL skips. */
int mpig_attn_read_cache(mpig_ctx *ctx, int layer, void *k_bf16, void *v_bf16, float *kn, void *stream);

/* ---- the GPU-side glue of LSHSparseAttnServer.decode ------------------------------------------ */
/* attnserver.py:264-270: codes int32 (B*Hq, L) of query bf16 (B*Hq, d); also writes
 * query_norm fp32 (B*Hq) = ||q||_2 in fp32 (attnserver.py:300) when non-NULL. */
int mpig_simhash(mpig_ctx *ctx, const void *query_bf16, int32_t *codes, float *query_norm, void *stream);
/* attnserver.py:142-153: the per-(request, kv-head) mean key (bf16 (Hkv, d)) and the sink+local
 * window rows of a sparse layer, keys ALREADY centred: k, v bf16 (Hkv, w, d). */
int mpig_window_fill(mpig_ctx *ctx, int layer, int request, const void *avg_k_bf16, const void *k_bf16,
                     const void *v_bf16, int w, void *stream);
/* LSHSparseAttnServer.plan (attnserver.py:196-224): advance every request's window length by one.  Refuses (MPIG_ESTATE) when a
 * window is full; mpig_spill_window between tokens frees it. */
int mpig_plan(mpig_ctx *ctx, void *stream);
/* Move the oldest non-sink rows of every request's sparse window into the sampled store (no reference equivalent; the
 * reference caps a generation at generation_buffer tokens).  For every request b and every sparse layer, window rows
 * [sink, win_len[b] - keep) become offloaded keys n_old .. n_old + g_b - 1 (records, key norms, and their codes merged into the
 * L hash tables), rows [win_len[b] - keep, win_len[b]) move down to [sink, sink + keep) and win_len[b] = sink + keep, with
 * g_b = max(0, win_len[b] - sink - keep), sink = num_sink_tokens and n_old the count mpig_attn_fill recorded plus earlier
 * spills (the tables must have been built over the same keys).  keep = num_local_tokens gives a layer the shape a prefill of
 * P + g tokens would have, centred with the prefill's mean key.  spilled_out int32 [B] (host, may be NULL) receives g_b.
 * Reads the device window lengths (synchronises `stream`), so it is correct after eager plan() calls and after replays of a
 * captured step alike.  Not capturable.  A decode step captured before a spill stays valid after it.  Dense layers are
 * untouched.  The spilled keys go into the store and tables of the request's slot: the requests of a slot spill into it in
 * request order, so n_old is the slot's count plus the rows of the slot's earlier requests.  The two modes differ in two ways
 * only.  Without shared spill (shared_spill = 0) a request with g_b > 0 must be alone on its slot among requests with a
 * non-empty window: a request that shares its context generates at most generation_buffer tokens.  In shared spill mode
 * several requests of a slot may spill, and each spilled key is private to its request.
 * MPIG_EINVAL: keep < 0 or sink + keep >= window capacity; MPIG_ESTATE: the slot's count plus all its requests' rows >
 * max_length for some sparse layer, a spilling request shares its slot with another request whose window is not empty (not in
 * shared spill mode), the sparse layers of a slot disagree on its private key count (shared spill mode, after a partial
 * refill), or no hash_func set.  On these errors nothing is modified. */
int mpig_spill_window(mpig_ctx *ctx, int keep, int32_t *spilled_out, void *stream);
/* Shared spill mode (shared_spill = 1): reclaim the dead private keys of context slot `slot` (-1: every slot).  A private key is
 * dead when no request sees it any more (vis[slot][p] == 0: its owner was forked over, reordered over, rebound or retired).
 * Every live private key keeps its time order and moves to the lowest free offset: live key j (ascending offsets) becomes
 * store index private_lo + j of every sparse layer, its record and key norm with it, vis[slot][j] takes its word (the words
 * past the live count become 0), the slot's key count drops by the number reclaimed, and the slot's tables become what a
 * build over the compacted keys would make (the live keys are rehashed with the spill's kernel, so their codes are the same).
 * Every request then samples exactly what it sampled before, up to that renumbering.  Windows, lengths, avg_k, dense layers
 * and the pending step are untouched; no array moves, so a step captured before the call stays valid after it.  reclaimed_out
 * int32 [C] (host, may be NULL) receives the keys removed per slot.  Without shared spill there are no private keys: zeros and
 * nothing launched.  Synchronises `stream`; not capturable.  Allocates scratch for the live keys of one layer (live x Hkv x
 * (2 d + 2 L) bytes) for the call.
 * MPIG_EINVAL: slot outside [-1, C); MPIG_ESTATE: the sparse layers of a slot disagree on its private key count (after a partial
 * refill), or no hash_func set; MPIG_ENOMEM: the scratch allocation failed.  On these errors nothing is modified. */
int mpig_compact_context(mpig_ctx *ctx, int slot, int32_t *reclaimed_out, void *stream);
/* Diagnostic accessor (the tests and scripts/compact_bench.py read the map through it; decoding never needs it).  Shared spill
 * mode: copy the visibility map (uint32 [C][max_length], bit b of word [c][p] = request b sees private key p of slot c) to the
 * device buffer vis_out.  MPIG_ESTATE without shared spill. */
int mpig_read_visibility(mpig_ctx *ctx, uint32_t *vis_out, void *stream);
/* Fused sparse-layer decode (attnserver.py:261-312): centre + append the new key/value to the
 * window, SimHash, probe, gather attention over window + sample with the LSE merge folded in -- one kernel launch.
 * query bf16 (B, Hq, d); key/value bf16 (B, Hkv, d); out bf16 (B, Hq*d).
 * Call mpig_plan once per token before the layers' decodes: the new row lands at window position win_len-1.  When the
 * window is full (see mpig_error_flags) the last row is overwritten. */
int mpig_decode(mpig_ctx *ctx, int layer, const void *query_bf16, const void *key_bf16,
                const void *value_bf16, void *out_bf16, void *stream);
/* Same call with HOST buffers: q/k/v are staged through one mapped pinned block that the kernels read directly and the
 * output is written straight back into it (no copy engine calls); returns after the stream drains. */
int mpig_decode_host(mpig_ctx *ctx, int layer, const void *query_bf16, const void *key_bf16,
                     const void *value_bf16, void *out_bf16, void *stream);
/* mpig_decode with a CUDA event between the three launches (SimHash+append | probe | attend).  The call does
 * NOT synchronise: the events of call number i since the last collect are kept in the context, so a whole
 * sequence of layers can be enqueued back to back (GPU kept busy, clocks steady) and read afterwards with
 * mpig_timing_collect, which synchronises and writes 3 floats (ms) per recorded call.  Measurement aid for
 * bench.py's roofline; not capturable, and the programmatic-dependent-launch overlap is off in this mode. */
int mpig_decode_timed(mpig_ctx *ctx, int layer, const void *query_bf16, const void *key_bf16,
                      const void *value_bf16, void *out_bf16, void *stream);
int mpig_timing_collect(mpig_ctx *ctx, float *stage_ms, int max_calls, int *n_calls);
/* Sample of the last mpig_decode, copied out of the context's scratch: nnz int32 (B*Hq) and, when
 * non-NULL, results int32 (B*Hq, M) (the arguments LSH::batch_retrieve fills, lsh.cc:210-216).  The fused decode keeps the
 * index list in shared memory; results are valid only if option "save_mask" was set before the decode. */
int mpig_last_probe(mpig_ctx *ctx, int32_t *nnz_out, int32_t *results_out, void *stream);
/* Query codes int32 (B*Hq, L) the last mpig_decode probed with (attnserver.py:264-270).  The fused decode keeps them in
 * shared memory: valid only if option "save_mask" was set before the decode. */
int mpig_last_codes(mpig_ctx *ctx, int32_t *codes_out, void *stream);
/* fp32 (B*Hq, d) attention output of the last mpig_decode / mpig_dense_decode / mpig_attention_wrapper before the bf16
 * rounding of the ABI (option "out_f32" must have been set before that call). */
int mpig_last_out_f32(mpig_ctx *ctx, float *out_f32, void *stream);
/* Clock stamps of the kernels' debug instantiations (options "attend_debug" / "fused_debug"): 16 uint64 per warp / per CTA,
 * copied to HOST memory. */
int mpig_debug_read(mpig_ctx *ctx, unsigned long long *host_out, int nwarps);
int mpig_fused_debug_read(mpig_ctx *ctx, unsigned long long *host_out, int nctas);

/* ---- verification steps of T tokens (speculative decoding; no reference equivalent) ------------------------------------------
 * A step checks T candidate tokens (1 <= T <= 8) of every request in one pass over the weights:
 *   mpig_plan_tokens(T) -> per layer mpig_decode_tokens / mpig_dense_decode_tokens(T) -> mpig_rewind(drop).
 * The layer appends the T new K/V rows of request b at positions base_b .. base_b + T - 1 (base_b = length before the plan) and
 * query token t attends causally: window / dense rows [0, base_b + t] and, on sparse layers, its own LSH sample (own codes, probe
 * and importance weights).  The result equals T single-token steps on the same inputs: identical codes, nnz and index sets, fp32
 * outputs equal up to summation order.  mpig_rewind then drops the last drop[b] of the T tokens of request b.  The tables and the
 * sampled store are never touched; mpig_spill_window keeps working because it reads the device lengths.
 *
 * Allocates the per-step scratch for up to t_max <= 8 tokens: query codes, norms, nnz, LSE pairs, the fp32 output copy and the
 * save_mask index lists / bitmaps grow from B*Hq to B*t_max*Hq rows.  Not capturable (allocates, synchronises the device).  The
 * scratch moves to new addresses, so the call is refused (MPIG_ESTATE) once a plan has been captured into a CUDA graph: reserve
 * before capturing.  Without it only T = 1 is accepted. */
int mpig_reserve_query_tokens(mpig_ctx *ctx, int t_max);
/* mpig_plan for a step of T tokens: every window and dense length advances by T.  T = 1 is exactly mpig_plan.  The host-mirror
 * checks of mpig_plan apply to +T and refuse (MPIG_ESTATE) before anything is modified; the device saturates and raises the same
 * mpig_error_flags bits.  Records T as the pending step size (host state, also when captured); MPIG_EINVAL for T outside
 * [1, reserved]. */
int mpig_plan_tokens(mpig_ctx *ctx, int T, void *stream);
/* Sparse layer, T tokens: query bf16 (B, T, Hq, d), key / value bf16 (B, T, Hkv, d), out bf16 (B, T, Hq*d).  T must equal the
 * pending T (MPIG_ESTATE).  T = 1 is mpig_decode (bitwise).  T > 1: one append launch for the T centred rows, then the T-token
 * instantiation of the fused kernel under PDL (B*T*Hq clusters, several waves where one does not hold them; shapes with one CTA
 * per head hash the B*T*Hq rows in the stand-alone SimHash kernel first).  MPIG_EUNSUPPORTED with decode_impl = 0 or a shape the
 * fused kernel does not take.  After a T > 1 call, mpig_last_probe / mpig_last_codes / mpig_last_out_f32 return B*T*Hq rows in
 * (b, t, h) order (size the buffers accordingly); after any single-token decode they return B*Hq rows as before. */
int mpig_decode_tokens(mpig_ctx *ctx, int layer, int T, const void *query_bf16, const void *key_bf16, const void *value_bf16,
                       void *out_bf16, void *stream);
/* Dense layer, same shapes: one append launch for the T rows, then one launch per (request, kv-group) in which the T*G query rows
 * share every fetched K|V record (dense KV bytes per step do not grow with T).  MPIG_EUNSUPPORTED for T*G > 32 or dense_impl = 0. */
int mpig_dense_decode_tokens(mpig_ctx *ctx, int layer, int T, const void *query_bf16, const void *key_bf16, const void *value_bf16,
                             void *out_bf16, void *stream);
/* Drop the last drop[b] tokens of the pending step of request b (drop: DEVICE int32 (B,), 0 <= drop[b] <= T): both lengths shrink by
 * drop[b]; stale rows past the length are overwritten by the next plan.  Capturable (acceptance can be decided on the GPU).  A
 * request whose drop is outside [0, T] is left untouched and raises mpig_error_flags bit 2.  At most one rewind per plan
 * (MPIG_ESTATE).  Outside a capture the call synchronises `stream` and checks the drops first: if one is outside [0, T] it raises
 * bit 2, changes no length and returns MPIG_EINVAL (the rewind may then be repeated with valid drops); otherwise it rewinds and
 * refreshes the host mirror of the lengths from the device.  mpig_clear forgets the pending step.  Refused (MPIG_ESTATE) after
 * mpig_plan_tree: dropping a suffix of a tree is meaningless. */
int mpig_rewind(mpig_ctx *ctx, const int32_t *drop, void *stream);

/* ---- token trees (speculative decoding with several candidates per position; no reference equivalent) ---------------------------
 *   mpig_plan_tree(T, parents) -> per layer mpig_decode_tokens / mpig_dense_decode_tokens(T) -> mpig_accept(nodes, count).
 * A step of T nodes (1 <= T <= the reserved t_max) takes per request b a parent array parents[b][0..T): parents[b][0] = -1 and
 * 0 <= parents[b][t] < t (topological order, node 0 is the root).  The T new rows are appended at base_b .. base_b + T - 1 in node
 * order, as for a chain.  Node t attends to the context rows [0, base_b), the rows of its ancestors, its own row and, on sparse
 * layers, its own LSH sample; rows of the other nodes of the step are invisible.  Per node, the result equals a chain step over the
 * node's root path: identical codes, nnz and index lists, fp32 outputs equal up to summation order.  A chain (parents[t] = t - 1) is
 * exactly mpig_plan_tokens.  RoPE positions are the caller's: node t sits at position base + depth(t).
 *
 * mpig_plan_tree does the work of mpig_plan_tokens(T) (same host-mirror checks, same device saturation bits), and its plan kernel
 * checks every request's tree and records the per-node ancestor masks and a copy of the parents in context scratch allocated at
 * create time (nothing moves after a capture; parents may be reused right after the call).  parents: DEVICE int32 (B, T).
 * Capturable: under capture a malformed tree makes that request a chain and raises mpig_error_flags bit 3.  Eager calls read the
 * parents back first: on a malformed tree they raise bit 3, change nothing and return MPIG_EINVAL.  MPIG_EINVAL for T outside
 * [1, reserved]. */
int mpig_plan_tree(mpig_ctx *ctx, int T, const int32_t *parents, void *stream);
/* Commit the root path nodes[b][0..count[b]) of the pending step of request b (nodes: DEVICE int32 (B, T), count: DEVICE int32 (B)).
 * A path is valid when 0 <= count[b] <= T, nodes[b][0] = 0 and parents[nodes[b][i]] = nodes[b][i-1].  Row base + nodes[b][i] moves
 * to base + i in every sparse layer's window (all kv-heads) and every dense layer's KV, in one launch, and both lengths become
 * base + count[b].  Works after mpig_plan_tokens / mpig_plan too (a chain prefix of count nodes equals mpig_rewind(T - count)).
 * Capturable (acceptance can be decided on the GPU): a bad path leaves that request untouched and raises bit 3.  Outside a capture
 * the call synchronises `stream` and checks the paths first: on a bad one it raises bit 3, changes nothing and returns MPIG_EINVAL
 * (the accept may then be repeated).  At most one rewind or accept per plan (MPIG_ESTATE).  Row accesses stay inside the window and
 * dense capacities even after a plan that saturated.  mpig_clear forgets the pending step. */
int mpig_accept(mpig_ctx *ctx, const int32_t *nodes, const int32_t *count, void *stream);

/* ---- chunk steps: a prompt chunk appended to running requests (follow-up turns, a question per forked request) ------------------
 *   mpig_reserve_chunk_tokens(t_max) once -> mpig_plan_chunk(T) -> per layer mpig_chunk_attend(T) -> [mpig_rewind(drop)]
 *   -> mpig_spill_window() before the window fills.
 * A chunk step appends the T new K/V rows of request b at base_b .. base_b + T - 1 of every layer (1 <= T <= t_max <= 1024), exactly
 * as a T-token verification step does (sparse layers centre the keys with avg_k, dense layers store them raw), and query token t
 * gets EXACT softmax attention (scale 1/sqrt(d); no sampling, no importance weights) over
 *   sparse layer: every key of the slot's sampled store the request sees (shared spill mode: the prompt keys and the
 *                 private keys it spilled or inherited) plus window rows [0, base_b + t];
 *   dense layer:  dense rows [0, base_b + t] (dense_tail_rows = R > 0: the slot's prompt rows below the request's dense base, then its
 *                 tail).
 * Store and window keys of a request carry the same -avg_k shift, to which softmax is invariant: the result is the attention a
 * prefill of the whole conversation computes, up to rounding.  mpig_rewind(drop) afterwards keeps T - drop[b] tokens of request b
 * (attention is causal: the kept tokens' outputs do not depend on the dropped ones); mpig_spill_window then folds the chunk into
 * the store and the tables, and ordinary decode steps continue.  mpig_accept refuses a chunk step; mpig_decode_tokens and
 * mpig_dense_decode_tokens refuse it too.  After mpig_chunk_attend, mpig_last_out_f32 returns B*T*Hq rows; mpig_last_probe and
 * mpig_last_codes refuse until the next decode (a chunk step has no LSH sample).
 *
 * Allocates the chunk scratch (key-split states, merge tickets; the out_f32 copy grows to B*t_max*Hq rows).  Like
 * mpig_reserve_query_tokens: not capturable (allocates, synchronises the device) and refused (MPIG_ESTATE) once a plan has been
 * captured into a CUDA graph.  MPIG_EINVAL for t_max outside [1, 1024].  mpig_get_info("chunk_tokens_max") reports t_max. */
int mpig_reserve_chunk_tokens(mpig_ctx *ctx, int t_max);
/* mpig_plan_tokens for a chunk step: every window and dense length advances by T, with the same host-mirror checks (T must fit the
 * window and the dense capacity, else MPIG_ESTATE and nothing changes) and the same device saturation bits.  Records the pending step
 * as a chunk step of T tokens.  Capturable.  MPIG_EINVAL for T outside [1, reserved]. */
int mpig_plan_chunk(mpig_ctx *ctx, int T, void *stream);
/* Sparse or dense layer, a chunk step of T tokens: query bf16 (B, T, Hq, d), key / value bf16 (B, T, Hkv, d), out bf16 (B, T, Hq*d),
 * rounded as the other attention outputs.  One append launch (the T-token verification step's), then the chunk attention kernel under
 * programmatic dependent launch (csrc/attend_chunk.cu, mma.sync tensor-core tiles); no host synchronisation.  Capturable for a fixed
 * T: a replay reads the lengths, bindings, store lengths and visibility maps of the replay.  MPIG_ESTATE when the pending step is not
 * a chunk step of this T (or a dense layer has no dense KV); MPIG_EINVAL for T outside [1, reserved]. */
int mpig_chunk_attend(mpig_ctx *ctx, int layer, int T, const void *query_bf16, const void *key_bf16, const void *value_bf16,
                      void *out_bf16, void *stream);

/* ---- prefill attention ---------------------------------------------------------------------------------------------------
 * Exact causal attention of a prompt chunk over its keys (flashinfer single_prefill_with_kv_cache, causal, NHD;
 * models/llama.py:250-257).  q bf16 (q_len, Hq, d), k/v bf16 (kv_len, Hkv, d) with the context's per-rank head counts;
 * query i sees keys [0, kv_len - q_len + i].  out bf16 (q_len, Hq, d); out_f32 (q_len, Hq, d) or NULL.  Reads and writes
 * no context state (any layer, any pending step); no host synchronisation; capturable.  csrc/attend_prefill.cu: wgmma
 * tensor-core tiles fed by TMA.  MPIG_EINVAL: q_len < 1, kv_len < q_len, a null input or output, or a base pointer that is not
 * 16-byte aligned; MPIG_EUNSUPPORTED: head_dim != 128 or Hq / Hkv outside [1, 8]. */
int mpig_prefill_attend(mpig_ctx *ctx, const void *q_bf16, const void *k_bf16, const void *v_bf16, int q_len, int kv_len,
                        void *out_bf16, float *out_f32, void *stream);

/* ---- dense layers (attnserver.py:116-120, 235-259), only with cfg.alloc_dense_kv -------------- */
/* k, v bf16 (P, Hkv, d) -- the prefill cache in NHD layout as models/llama.py:282 passes it. */
int mpig_dense_fill(mpig_ctx *ctx, int layer, int request, const void *k_bf16, const void *v_bf16,
                    int seq_len, void *stream);
/* Single-token dense decode.  MPIG_EUNSUPPORTED for G = Hq / Hkv > 32 with dense_impl = 1. */
int mpig_dense_decode(mpig_ctx *ctx, int layer, const void *query_bf16, const void *key_bf16,
                      const void *value_bf16, void *out_bf16, void *stream);

/* ---- exchange step of KV-head tensor parallelism over NVLink peer memory (peer.cu) ------------------------------------------
 * The path shards by KV head (evaluations/RULER/pred/attnserver_dist.py:252-254) with no exchange inside SimHash / probe /
 * attention.  What the caller's TP layout exchanges per layer -- the all-gather of head outputs of the north-star layout, or the
 * two all-reduces of llama_dist.py:209,218 -- is 8-16 KB: pure latency.  A mpig_peer is one cudaMalloc'ed exchange block per
 * rank, mapped into every other rank through CUDA IPC; a collective is ONE kernel launch: 16-byte stores of {word, flag, word,
 * flag} lines into the peers' blocks (the payload carries its own arrival flag: no fence, no atomic) and a spin on the lines of
 * the consumer's own block.  No NCCL, no host, CUDA-graph capturable.
 *   1. every rank: mpig_peer_create, mpig_peer_handle (64 bytes) -> exchange the handles out of band (torch.distributed)
 *   2. every rank: mpig_peer_connect(all handles in rank order); barrier
 * slot_bytes >= the largest payload of one rank (multiple of 16).  All ranks must issue the same sequence of collectives. */
typedef struct mpig_peer mpig_peer;
int mpig_peer_create(mpig_ctx *ctx, int rank, int world, size_t slot_bytes, mpig_peer **out);
int mpig_peer_handle(mpig_peer *p, void *handle_out_64_bytes);
int mpig_peer_connect(mpig_peer *p, const void *handles_world_x_64_bytes);
void mpig_peer_destroy(mpig_peer *p);
/* src (bytes) of every rank -> dst (world x bytes) in rank order on every rank */
int mpig_peer_all_gather(mpig_peer *p, const void *src, void *dst, size_t bytes, void *stream);
/* in-place sum over ranks of n bf16 elements: fp32 accumulation in rank order, one rounding (bitwise identical on all ranks) */
int mpig_peer_all_reduce_bf16(mpig_peer *p, void *buf, size_t n, void *stream);
/* mpig_decode whose EPILOGUE is the all-gather: each head's output row is stored from the attention kernel straight into every
 * rank's gather slot (no separate exchange kernel on the producer side); gathered = (world, B*Hq_loc*d) bf16 in rank order. */
int mpig_decode_allgather(mpig_ctx *ctx, mpig_peer *p, int layer, const void *query_bf16, const void *key_bf16,
                          const void *value_bf16, void *out_local_bf16, void *gathered_bf16, void *stream);
/* Every spin on a line is bounded (~2 s): number of lines a collective gave up on (a dead peer); 0 on a healthy run. */
int mpig_peer_timeouts(mpig_peer *p, unsigned long long *count);
/* consumer half alone (after a producer kernel stored the lines; `parts` is ignored: arrival is per line) */
int mpig_peer_wait_gather(mpig_peer *p, void *dst, size_t bytes, int parts, void *stream);

/* ---- launch accounting (bench.py's gpu_launches) ---------------------------------------------- */
/* number of kernels this library has launched on behalf of `ctx` since creation */
uint64_t mpig_launch_count(const mpig_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* MAGICPIG_B200_H */
