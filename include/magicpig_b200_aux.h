/*
 * magicpig_b200_aux.h -- caller-side helpers used by the benchmark harness (magicpig_b200/llama_runner.py).
 *
 * NOT part of the drop-in boundary (that is magicpig_b200.h).  These fused elementwise kernels and the decode GEMV stand in for
 * the small torch/FlashInfer ops the reference's CALLER runs around the attention server every layer
 * (models/utils.py: layer_norm -> flashinfer.rmsnorm :46-55, apply_rotary_pos_emb :36-44; models/llama.py:
 * residual adds :210-218, silu(gate)*up :171-181), so that the decode step is not dominated by ~20 tiny launches per
 * layer.  Device pointers, bf16, explicit stream, int status like the main ABI.
 */
#ifndef MAGICPIG_B200_AUX_H
#define MAGICPIG_B200_AUX_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* h (rows, hidden) bf16 += delta (rows, hidden) bf16 [delta may be NULL]; x_out = rmsnorm(h) * weight.  hidden % 8 == 0. */
int mpig_aux_add_rmsnorm(void *h_inout, const void *delta, const void *weight, float eps, void *x_out, int rows, int hidden,
                         void *stream);
/* qkv (B, (Hq+2*Hkv)*d) bf16 -> q_out (B,Hq,d), k_out (B,Hkv,d) with rotate-half RoPE at position pos[b], v_out (B,Hkv,d).
 * cos/sin: (max_pos, d) bf16 tables; pos: (B) int64.  d == 128. */
int mpig_aux_rope_split(const void *qkv, const void *cos_tab, const void *sin_tab, const int64_t *pos, void *q_out, void *k_out,
                        void *v_out, int B, int Hq, int Hkv, void *stream);
/* gate_up (rows, 2*inter) bf16 -> out (rows, inter) = silu(gate) * up.  inter % 8 == 0. */
int mpig_aux_silu_mul(const void *gate_up, void *out, int rows, int inter, void *stream);

/* y (rows, N) bf16 = x (rows, K) bf16 . weight^T, weight (N, K) row-major bf16 as torch.nn.Linear stores it, fp32
 * accumulation; rows <= 8 (decode batch), K % 256 == 0, rows*K*2 <= 200 KB.  A weight-streaming GEMV: stands in for the
 * library GEMM of the model's linear layers (models/llama.py:195-218) at decode batch sizes.
 * swiglu != 0: weight is [gate (N rows); up (N rows)] and y = silu(x.gate^T) * (x.up^T)  (models/llama.py:171-181). */
int mpig_aux_gemv(const void *weight, const void *x, void *y, int rows, int N, int K, int swiglu, void *stream);
/* Same with the residual add + RMSNorm folded into the prologue: x = rmsnorm(h_in + delta) * ln_weight (delta may be NULL),
 * h_out = h_in + delta (a DIFFERENT buffer: every CTA re-reads h_in, so the residual stream is ping-ponged), K = hidden. */
int mpig_aux_norm_gemv(const void *weight, const void *h_in, const void *delta, const void *ln_weight, float eps, void *h_out,
                       void *y, int rows, int N, int K, int swiglu, void *stream);
/* Prologue as above, weight = [q heads; k heads; v heads] ((Hq + 2*Hkv) * 128 rows), and the epilogue of
 * mpig_aux_rope_split: q_out (rows, Hq, 128), k_out (rows, Hkv, 128) rotated at pos[row], v_out copied. */
int mpig_aux_norm_qkv_rope(const void *wqkv, const void *h_in, const void *delta, const void *ln_weight, float eps, void *h_out,
                           const void *cos_tab, const void *sin_tab, const int64_t *pos, void *q_out, void *k_out, void *v_out,
                           int rows, int Hq, int Hkv, int K, void *stream);

/* Programmatic dependent launch on the two edges around the attention kernel (process-wide switch, default 0 = off):
 * bit 0: mpig_aux_norm_qkv_rope triggers the launch of its successor (the fused attention kernel) at its top, so that kernel's
 * launch latency and constant-data prologue overlap the projection's tail; bit 1: mpig_aux_gemv (non-SwiGLU) is launched as a
 * programmatic dependent and waits for its producer before reading x (the o-projection parks behind the attention kernel).
 * Returns the previous mask. */
int mpig_aux_set_pdl(int mask);

/* One token for each of B rows of fp32 logits (B, V), row stride ld >= V: temperature / top-p sampling as the reference's
 * caller does it (models/utils.py:57-100, topp_temperature_decode; argmax when the temperature is small).  Contract, row b,
 * logits l_i, T = temperature[b], p = top_p[b] (device fp32 (B,) each, so a captured call picks up new values):
 *   - T <= 0 (or NaN): greedy, the smallest i with l_i == max l (torch.argmax's first occurrence).
 *   - T > 0: w_i = exp2f((l_i - m) * (1.44269504f / T)) in fp32, m = max l, -inf logits weigh 0; W_i = floor(w_i * 2^40) as a
 *     u64, S = sum W_i.  Token i is kept iff the W of the tokens before it in the order (W descending, lower index first on
 *     ties) sum to <= floor(p * S), computed exactly (p >= 1 keeps all, p <= 0 only the first).  r = the first 64 bits of
 *     Philox4x32-10 (curand_Philox4x32_10, counter (*offset lo, *offset hi, b, 0), key (seed lo, seed hi)); target =
 *     umulhi64(r, S_keep); the token is the kept index, in index order, at which the running kept sum first exceeds target.
 *     Bitwise deterministic: everything after the fp32 weights is integer.
 *   - a row with a NaN or +inf logit, or with no finite logit, gets token 0 and sets bit b % 32 of status[b / 32] (status may be
 *     NULL; never cleared here).
 * offset: device u64, read and never written (the caller advances it, e.g. in the same graph).  Optional bookkeeping:
 *   ids_out (int64, may be NULL): ids_out[b * ids_stride] = token.
 *   tokens_out (int32 (B, max_new), may be NULL; needs count and done, int32 (B,)): unless done[b], append the token at
 *   count[b] and increment it; done[b] = 1 when the token is one of the n_eos <= 8 ids eos_ids (a HOST array) or count[b]
 *   reaches max_new.
 *   debug (int64 (B, 5), may be NULL): S, floor(p * S), S_keep, kept count, target (greedy rows: 0, 0, 0, 1, 0; invalid rows:
 *   zeros).  debug_w (fp32 (B, V), may be NULL): the weights w_i of the rows with T > 0.
 * One cluster of C <= 8 CTAs per row, C = ceil(V / 4096) (V up to 409 600).  Refused with MPIG_EINVAL: B < 1, V < 1, V beyond
 * that, ld < V, null or misaligned logits, null temperature / top_p / offset, n_eos > 8, tokens_out without count / done.
 * Capturable. */
int mpig_aux_sample(const float *logits, int B, int V, int64_t ld, const float *temperature, const float *top_p, uint64_t seed,
                    const uint64_t *offset, int64_t *ids_out, int64_t ids_stride, int32_t *tokens_out, int32_t *count,
                    int32_t *done, int max_new, const int32_t *eos_ids, int n_eos, int32_t *status, int64_t *debug,
                    float *debug_w, void *stream);
/* Clusters of mpig_aux_sample's kernel at vocabulary size V that the current device keeps resident at once. */
int mpig_aux_sample_occupancy(int V, int *clusters);

/* Speculative sampling: the acceptance of a verification step's draft tokens and the next token, for B requests in one call.
 * logits: fp32 rows (b, t) at logits + b * ld_b + t * ld_t, t < T (1 <= T <= 8), the logits after each of the step's T input
 * tokens; ids: int64 rows at ids + b * ids_stride, the step's inputs, so request b's drafts are ids[b, 1 .. T-1].  Row (b, t) is
 * sampled with exactly mpig_aux_sample's rule (same w_i, W_i, nucleus, S_keep; temperature[b], top_p[b], seed, *offset).
 * For t <= T - 2 let d = ids[b, t + 1] (an id outside [0, V) is never accepted):
 *   - greedy (T <= 0): d is accepted iff it is the row's first argmax.
 *   - sampled: d is accepted iff it is kept and umulhi64(r_acc, S_keep) < W_d, r_acc = the first 64 bits of Philox4x32-10 at
 *     counter (*offset lo, *offset hi, b, t + 1) under mpig_aux_sample's key: probability p(d), the nucleus probability of d.
 * k = the first row whose draft is rejected (T - 1 if all are accepted).  The request emits d_1 .. d_k, then one final token
 * from row k: rejected there, greedy -> the row's argmax; sampled -> a draw from the residual, the kept set without d, of mass
 * S_keep - W_d (S_keep when d is not kept), with mpig_aux_sample's counter (.., b, 0) and index-order scan skipping d; all
 * accepted -> mpig_aux_sample's draw on row T - 1.  Each emitted token then follows the nucleus distribution of its row given its
 * prefix (the standard rule for a deterministic, one-hot draft; it is NOT exact for drafts drawn from a draft distribution).
 * At T = 1 the token is mpig_aux_sample's, bit for bit.  A row with a NaN or +inf logit, or no finite one, accepts nothing; if it
 * is row k the final token is 0 and bit b % 32 of status[b / 32] is set (status may be NULL).
 * Outputs: ids[b, 0] = the final token; drop[b] = T - 1 - k (int32 (B,), the mpig_rewind input; may be NULL; see below for a
 * request that ends).  rows: int32
 * (B, T, 2) scratch (each row's final token and flags).  Optional bookkeeping as mpig_aux_sample's, on a token history:
 * history int32 (B, history_ld) with length / limit / done int32 (B,): the emitted tokens are appended in order at length[b]
 * while length[b] < min(limit[b], history_ld); an EOS id (n_eos <= 8, host array; kept) or reaching the limit sets done[b] and ends
 * the appending.  A request that ends in the call after appending j tokens gets drop[b] = T - j, so it keeps only the rows of the
 * tokens it emitted before its last one.  A request with done[b] already set appends nothing, counts nothing and gets
 * drop[b] = T (its whole step is rewound).  steps / accepted int32 (B,) (both or neither): += 1 and += k per call for requests not done.  debug int64 (B, T, 9):
 * per row mpig_aux_sample's five integers (target = umulhi64(r, S_keep) of its draw), W_d, d's keep bit, umulhi64(r_acc, S_keep)
 * and the residual mass (greedy rows: 0 0 0 1 0 0 accept 0 0; invalid rows: zeros); debug_w fp32 (B, T, V): the weights.
 * Two launches: one cluster per row (mpig_aux_sample's kernel), then one thread per request.  Refused with MPIG_EINVAL: T outside
 * [1, 8], V as for mpig_aux_sample, ld_t < V or ld_b < (T - 1) ld_t + V, null or misaligned logits / ids / rows / temperature /
 * top_p / offset, ids_stride < T, n_eos > 8, history without length / limit / done, misaligned optional outputs.  Capturable. */
int mpig_aux_verify_sample(const float *logits, int B, int T, int V, int64_t ld_b, int64_t ld_t, const float *temperature,
                           const float *top_p, uint64_t seed, const uint64_t *offset, int64_t *ids, int64_t ids_stride,
                           int32_t *rows, int32_t *drop, int32_t *history, int64_t history_ld, int32_t *length, const int32_t *limit,
                           int32_t *done, int32_t *steps, int32_t *accepted, const int32_t *eos_ids, int n_eos, int32_t *status,
                           int64_t *debug, float *debug_w, void *stream);

/* Sampling filters: top-k, min-p and repetition / presence / frequency penalties, for the two calls below.  The arrays are device
 * arrays of shape (B,), so a captured call picks up new values:
 *   top_k              int32  off when <= 0
 *   min_p              fp32   in [0, 1]; off when 0 (NaN or <= 0 is off, > 1 is taken as 1)
 *   repetition_penalty fp32   r > 0; off when 1 (non-finite or <= 0 is taken as 1)
 *   presence_penalty   fp32   pr in [-2, 2]; off when 0 (non-finite is taken as 0)
 *   frequency_penalty  fp32   f in [-2, 2]; off when 0 (non-finite is taken as 0)
 * table: uint32 (B, ld), ld >= V, row b for request b: the low 31 bits of entry i are c_i, the times request b has emitted token i;
 * bit 31 is set when token i occurs in the request's prompt.  As in Hugging Face and vLLM, the repetition penalty applies to prompt
 * and output tokens, the presence and frequency penalties to output tokens only.
 * The rule for row b, raw logit l_i:
 *   1. penalties, fp32, every operation rounded to nearest with no contraction: seen_i = prompt bit or c_i > 0;
 *      l1 = seen_i ? (l > 0 ? l / r : l * r) : l;  l2 = l1 - f * (float)c_i;  l3 = c_i > 0 ? l2 - pr : l2.  A row whose three
 *      penalties are all neutral skips them (l3 = l).  Verification row t counts the drafts d_1 .. d_t of its step in c_i and
 *      seen_i: the tokens that row's prefix emits.  A NaN or +inf raw or penalised logit makes the row invalid (token 0, status).
 *   2. greedy (temperature <= 0): the first argmax of l3; top_k, min_p and top_p do not apply.
 *   3. w, W and S from l3 exactly as in mpig_aux_sample.
 *   4. truncation, in Hugging Face's processor order, each set a prefix of the order (W descending, lower index first on ties):
 *      top-k: n_k = min(top_k, V) if top_k > 0 else V, S_k = the mass of the first n_k tokens;  top-p over the top-k set: order
 *      position j < n_k is kept iff the mass before it is <= floor(p * S_k) (computed as mpig_aux_sample computes floor(p * S));
 *      min-p: W_i >= floor(min_p * 2^40), computed the same way (the max has W = 2^40, so it always stays).  The kept set is the
 *      first K = max(1, min(n_k, n_p, n_m)) tokens of the order; S_keep, the draw, the draft acceptance and the residual work as in
 *      the unfiltered calls on that set.  With every filter neutral the result equals the unfiltered call's bit for bit.
 *   5. bookkeeping: the call increments the table entry of each token it appends (to tokens_out, or to the history), in the same
 *      call.  Rejected drafts and requests already done count nothing, and a call that appends nothing leaves the table as it is.
 * With one-hot drafts every token a verification step emits then follows the filtered distribution given the request's whole prefix. */
typedef struct mpig_sample_filters {
    const int32_t *top_k;
    const float *min_p;
    const float *repetition_penalty;
    const float *presence_penalty;
    const float *frequency_penalty;
    uint32_t *table;
    int64_t ld;
} mpig_sample_filters;

/* mpig_aux_sample with the filters above.  debug int64 (B, 8): mpig_aux_sample's five integers (floor(p * S_k) in place of
 * floor(p * S), the kept count K), then n_k, S_k and n_m, the tokens with W >= floor(min_p * 2^40) (greedy and invalid rows: zeros
 * there); debug_w: the weights of the penalised logits.  Refused with MPIG_EINVAL as mpig_aux_sample, and for a null filters, a
 * null or misaligned member, ld < V.  Capturable. */
int mpig_aux_sample_filtered(const float *logits, int B, int V, int64_t ld, const float *temperature, const float *top_p,
                             uint64_t seed, const uint64_t *offset, int64_t *ids_out, int64_t ids_stride, int32_t *tokens_out,
                             int32_t *count, int32_t *done, int max_new, const int32_t *eos_ids, int n_eos, int32_t *status,
                             int64_t *debug, float *debug_w, const mpig_sample_filters *filters, void *stream);
/* mpig_aux_verify_sample with the filters above; debug int64 (B, T, 12): the nine integers, then n_k, S_k and n_m.  Refused as
 * mpig_aux_verify_sample and mpig_aux_sample_filtered.  Capturable. */
int mpig_aux_verify_sample_filtered(const float *logits, int B, int T, int V, int64_t ld_b, int64_t ld_t, const float *temperature,
                                    const float *top_p, uint64_t seed, const uint64_t *offset, int64_t *ids, int64_t ids_stride,
                                    int32_t *rows, int32_t *drop, int32_t *history, int64_t history_ld, int32_t *length,
                                    const int32_t *limit, int32_t *done, int32_t *steps, int32_t *accepted, const int32_t *eos_ids,
                                    int n_eos, int32_t *status, int64_t *debug, float *debug_w, const mpig_sample_filters *filters,
                                    void *stream);

/* Prompt-lookup drafts: for request b with history h = history[b, 0 .. n) (int32 (B, ld), n = min(length[b], ld), device), write
 * T - 1 drafts into ids[b * ids_stride + 1 .. T - 1] (int64).  For each end e in [0, n - 2], m(e) = the largest m <= g_max with
 * h[e - i] == h[n - 1 - i] for all i < m; e* maximises (m(e), e) among m(e) >= g_min (the longest match, then the most recent);
 * draft i = h'[e* + 1 + i] with h' = h followed by the drafts (an overlapping copy: periodic text continues its period).  No
 * match: every draft is h[n - 1] (0 when n = 0).  One cluster of 8 CTAs per request, a max of (m << 32 | e), so deterministic.
 * Refused with MPIG_EINVAL: B < 1, T outside [1, 8], not 1 <= g_min <= g_max <= 8, null or misaligned pointers, ids_stride < T.
 * Capturable. */
int mpig_aux_ngram_draft(const int32_t *history, int B, int64_t ld, const int32_t *length, int64_t *ids, int64_t ids_stride, int T,
                         int g_min, int g_max, void *stream);

#ifdef __cplusplus
}
#endif
#endif
