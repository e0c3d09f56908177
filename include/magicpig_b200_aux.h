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

#ifdef __cplusplus
}
#endif
#endif
