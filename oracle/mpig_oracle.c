/*
 * mpig_oracle.c -- CPU restatement of MagicPIG's LSH-sampled sparse-attention decode path.
 *
 * TEST INFRASTRUCTURE ONLY.  This file is the parity checker for the CUDA kernels in
 * magicpig_b200/csrc/.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load it.  The product path never calls into oracle/.
 *
 * Parity status: PINNED.  tests/test_oracle_cpu.py checks every function here against
 *   (1) the unmodified reference operators compiled from a reference checkout into oracle/_ref/
 *       (oracle/build_ref.py), when those binaries are present, and
 *   (2) the committed golden vectors under tests/golden/ that were produced by running
 *       those reference binaries (tests/golden/make_golden.py).
 *
 * Plain scalar C, single threaded, one function per reference function.  Each function
 * cites the reference file:line it restates (paths relative to the reference repository).
 *
 * Build: gcc -O2 -shared -fPIC -o oracle/_build/libmpig_oracle.so oracle/mpig_oracle.c -lm
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif
#ifndef M_LOG2E
#define M_LOG2E 1.4426950408889634074
#endif

/* bf16 <-> fp32.  Widening is a 16-bit shift (FbgemmBfloat16ConvertAvx512.cc:36-43).
 * Narrowing in the reference's output path is "add 2^15, shift right 16"
 * (FbgemmBfloat16ConvertAvx512.cc:20-26): round-half-UP on the magnitude bits, not RNE. */
static inline float bf16_to_f32(uint16_t h) {
    uint32_t u = ((uint32_t)h) << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}
static inline uint16_t f32_to_bf16_half_up(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    return (uint16_t)((u + 0x8000u) >> 16);
}
/* torch's bf16 rounding (round-to-nearest-even), used where the reference rounds on the
 * GPU with torch ops (models/attnserver.py:265-266). */
static inline uint16_t f32_to_bf16_rne(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40u); /* NaN */
    uint32_t lsb = (u >> 16) & 1u;
    return (uint16_t)((u + 0x7fffu + lsb) >> 16);
}

uint16_t orc_f32_to_bf16_half_up(float f) { return f32_to_bf16_half_up(f); }
uint16_t orc_f32_to_bf16_rne(float f) { return f32_to_bf16_rne(f); }

/* ------------------------------------------------------------------------------------------
 * Stage 1: SimHash of the decode queries.       models/attnserver.py:264-270 (+ :55-57)
 *   norm_q = q / ||q||_2           (bf16 tensor ops: the norm and the quotient are each
 *                                   rounded to bf16, RNE)
 *   proj   = norm_q @ hash_func    (bf16 GEMM, fp32 accumulate; only the sign is used)
 *   code[h,l] = sum_{i<K} [proj[h, l*K+i] > 0] * 2^i
 * hash_func is (d, K*L) row-major bf16.  min_abs_proj (optional, per (h,l)) returns the
 * smallest |proj| among the K bits of that code, so a test can ignore bits whose sign is
 * decided by accumulation order.
 * ------------------------------------------------------------------------------------------ */
void orc_simhash(const uint16_t *q_bf16, /* (H, d) */
                 const uint16_t *hash_func_bf16, /* (d, K*L) */
                 int H, int d, int K, int L,
                 int32_t *codes, /* (H, L) out */
                 float *min_abs_proj /* (H, L) out, may be NULL */) {
    const int KL = K * L;
    float *nq = (float *)malloc(sizeof(float) * (size_t)d);
    for (int h = 0; h < H; ++h) {
        const uint16_t *q = q_bf16 + (size_t)h * d;
        /* torch.norm on a bf16 tensor accumulates in fp32 and rounds the result to bf16 */
        float ss = 0.f;
        for (int i = 0; i < d; ++i) {
            float v = bf16_to_f32(q[i]);
            ss += v * v;
        }
        float nrm = bf16_to_f32(f32_to_bf16_rne(sqrtf(ss)));
        for (int i = 0; i < d; ++i) nq[i] = bf16_to_f32(f32_to_bf16_rne(bf16_to_f32(q[i]) / nrm));
        for (int l = 0; l < L; ++l) {
            int32_t code = 0;
            float mn = INFINITY;
            for (int i = 0; i < K; ++i) {
                const int col = l * K + i; /* table-major columns, little-endian bits (:268-270) */
                double acc = 0.0;
                for (int k = 0; k < d; ++k) acc += (double)nq[k] * (double)bf16_to_f32(hash_func_bf16[(size_t)k * KL + col]);
                if (acc > 0.0) code |= (1 << i);
                float a = (float)fabs(acc);
                if (a < mn) mn = a;
            }
            codes[(size_t)h * L + l] = code;
            if (min_abs_proj) min_abs_proj[(size_t)h * L + l] = mn;
        }
    }
    free(nq);
}

/* ------------------------------------------------------------------------------------------
 * Table storage + build from sorted codes.       library/lsh/lsh.cc:143-201 (LSH::fill)
 *   table_start/table_end : int32 [Hkv][L][NB]   (must be zero on entry, lsh.cc:179)
 *   table                 : int32 [Hkv][L][max_length], first n of each row valid
 * for one (layer, request).  sorted_codes int16 (Hkv,L,n), sorted_indices int32 (Hkv,L,n).
 * ------------------------------------------------------------------------------------------ */
void orc_lsh_fill(const int16_t *sorted_codes, const int32_t *sorted_indices,
                  int Hkv, int L, int n, int NB, int max_length,
                  int32_t *table_start, int32_t *table_end, int32_t *table) {
    for (int i = 0; i < Hkv; ++i)
        for (int j = 0; j < L; ++j) {
            const int16_t *v = sorted_codes + ((size_t)i * L + j) * n;
            int32_t *ms = table_start + ((size_t)i * L + j) * NB;
            int32_t *me = table_end + ((size_t)i * L + j) * NB;
            for (int k = 0; k < n; ++k) { /* lsh.cc:177-186 */
                const int c = (int)v[k];
                if (me[c] == 0) {
                    ms[c] = k;
                    me[c] = k + 1;
                } else {
                    me[c] += 1;
                }
            }
            memcpy(table + ((size_t)i * L + j) * max_length, sorted_indices + ((size_t)i * L + j) * n,
                   sizeof(int32_t) * (size_t)n); /* lsh.cc:197-200 */
        }
}

/* ------------------------------------------------------------------------------------------
 * Stage 2: probe.     library/lsh/lsh.cc:243-288 (LSH::retrieve), :210-241 (batch_retrieve)
 * For q-head `head` (kv group = head / G): walk the L buckets named by the query codes,
 * bump a saturating per-key byte 0->1->2 and emit the key index on the 1->2 transition.
 * Output order = second-hit order (unspecified by the reference's tests; compare as sets).
 * mask (uint8 [H][max_length]) is the reference's scratch (= get_mask(), lsh.cc:308-314).
 * ------------------------------------------------------------------------------------------ */
static int orc_retrieve_one(const int32_t *table_start, const int32_t *table_end, const int32_t *table,
                            int L, int NB, int max_length, int G, int head, const int32_t *query,
                            int32_t *results, uint8_t *mask) {
    const int g = head / G; /* lsh.cc:251 */
    const int32_t *start = table_start + (size_t)g * L * NB;
    const int32_t *end = table_end + (size_t)g * L * NB;
    const int32_t *content = table + (size_t)g * L * max_length;
    const int32_t *q = query + (size_t)head * L;
    int32_t *res = results + (size_t)head * max_length;
    uint8_t *m = mask + (size_t)head * max_length;
    memset(m, 0, (size_t)max_length); /* lsh.cc:260 */
    int cnt = 0;
    for (int i = 0; i < L; ++i) {
        const int b = q[i];
        const int s = start[(size_t)i * NB + b], e = end[(size_t)i * NB + b];
        const int32_t *c = content + (size_t)i * max_length;
        for (int j = s; j < e; ++j) { /* lsh.cc:272-283 */
            const int idx = c[j];
            const uint8_t mv = m[idx];
            if (mv == 0)
                m[idx] = 1;
            else if (mv == 1) {
                m[idx] = 2;
                res[cnt++] = idx;
            }
        }
    }
    return cnt;
}

void orc_lsh_batch_retrieve(const int32_t *table_start, const int32_t *table_end, const int32_t *table,
                            int L, int NB, int max_length, int G, int H_total, /* = B*Hq */
                            const int32_t *query, int32_t *results, int32_t *nnz, uint8_t *mask) {
    for (int h = 0; h < H_total; ++h)
        nnz[h] = orc_retrieve_one(table_start, table_end, table, L, NB, max_length, G, h, query, results, mask);
}

/* Independent restatement of the SELECTION RULE straight from unsorted key codes
 * (library/lsh/test.py:43: (hash_code == query).sum(dim=1) > 1): full collision counts.
 * key_codes int16 (Hkv_total, L, n); counts int32 (H_total, n) out. */
void orc_collision_counts(const int16_t *key_codes, int L, int n, int G, int H_total,
                          const int32_t *query, int32_t *counts) {
    for (int h = 0; h < H_total; ++h) {
        const int g = h / G;
        int32_t *c = counts + (size_t)h * n;
        memset(c, 0, sizeof(int32_t) * (size_t)n);
        for (int l = 0; l < L; ++l) {
            const int16_t *kc = key_codes + ((size_t)g * L + l) * n;
            const int qc = query[(size_t)h * L + l];
            for (int j = 0; j < n; ++j) c[j] += (kc[j] == qc);
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * Stage 3: gather attention for ONE q-head.   library/sparse_attention/sparse_attention.cc
 *   qk_kernel :38-67 / qk_kernel_bf16_impl :69-103      s_j = q . K[ind_j]      (fp32)
 *   transform_kernel :164-184                            LSH-probability re-weighting
 *   softmax_kernel :186-240                              p_j, base-2 LSE
 *   wv_kernel :321-347                                   o = sum_j p_j V[ind_j]  -> bf16
 * query is bf16 (the AVX512_BF16 route, :694-745, takes the bf16 query as is; the fp32 route
 * widens it exactly, :880) -- both see the same real numbers.
 * score (nnz floats, may be NULL) receives the normalised probabilities (= get_score()).
 * nnz == 0: reference yields lse = -inf and an untouched/zero output (SURVEY 7.3 #7).
 * ------------------------------------------------------------------------------------------ */
void orc_attention_head(const uint16_t *key /* [max_length][d] bf16 */, const uint16_t *value,
                        const float *key_norm /* [max_length] */, int d, int K, int L,
                        const uint16_t *q_bf16 /* [d] */, float q_norm, const int32_t *ind, int nnz,
                        uint16_t *out_bf16 /* [d] */, float *max_value, float *expsum, float *score) {
    float *s = (float *)malloc(sizeof(float) * (size_t)(nnz > 0 ? nnz : 1));
    const float sqrt_dim = sqrtf((float)d);
    if (nnz <= 0) {
        for (int i = 0; i < d; ++i) out_bf16[i] = 0;
        *max_value = -INFINITY;
        *expsum = -INFINITY;
        free(s);
        return;
    }
    for (int j = 0; j < nnz; ++j) { /* qk */
        const uint16_t *k = key + (size_t)ind[j] * d;
        double acc = 0.0;
        for (int i = 0; i < d; ++i) acc += (double)bf16_to_f32(q_bf16[i]) * (double)bf16_to_f32(k[i]);
        s[j] = (float)acc;
    }
    for (int j = 0; j < nnz; ++j) { /* transform_kernel :173-183, same expression types */
        float norm = q_norm * key_norm[ind[j]];
        float theta = acosf(s[j] / norm);
        float proba = (float)(1 - theta / M_PI);
        float p = powf(proba, (float)K);
        float qq = 1 - p;
        float w = 1 - powf(qq, (float)(L - 1)) * (L * p + qq);
        s[j] = (float)(s[j] / sqrt_dim - logf((float)(w + 1e-4)));
    }
    float m = s[0]; /* softmax_kernel :195-239 (libm expf everywhere; the reference uses a
                       3rd-order 2^x polynomial for full 16-lane groups, rel. err ~1e-4) */
    for (int j = 1; j < nnz; ++j)
        if (s[j] > m) m = s[j];
    float sum = 0.f;
    for (int j = 0; j < nnz; ++j) {
        s[j] = expf(s[j] - m);
        sum += s[j];
    }
    for (int j = 0; j < nnz; ++j) s[j] /= sum;
    *max_value = (float)(m * M_LOG2E);
    *expsum = log2f(sum) + *max_value;
    float *o = (float *)calloc((size_t)d, sizeof(float)); /* wv :329-345 */
    for (int j = 0; j < nnz; ++j) {
        const uint16_t *v = value + (size_t)ind[j] * d;
        for (int i = 0; i < d; ++i) o[i] = fmaf(bf16_to_f32(v[i]), s[j], o[i]);
    }
    for (int i = 0; i < d; ++i) out_bf16[i] = f32_to_bf16_half_up(o[i]);
    if (score) memcpy(score, s, sizeof(float) * (size_t)nnz);
    free(o);
    free(s);
}

/* attention_wrapper for all B*Hq heads (sparse_attention.cc:867-925 loop structure).
 * key/value: bf16 [B*Hkv][max_length][d]; key_norm fp32 [B*Hkv][max_length];
 * max_value_expsum: fp32 (2, H_total): row 0 = m*log2e, row 1 = LSE2. */
void orc_attention_wrapper(const uint16_t *key, const uint16_t *value, const float *key_norm,
                           int d, int max_length, int G, int H_total, int K, int L,
                           const uint16_t *q_bf16, const float *q_norm, const int32_t *ind, const int32_t *nnz,
                           uint16_t *out_bf16, float *max_value_expsum, float *score /* (H_total,max_length) or NULL */) {
    for (int h = 0; h < H_total; ++h) {
        const int g = h / G;
        orc_attention_head(key + (size_t)g * max_length * d, value + (size_t)g * max_length * d,
                           key_norm + (size_t)g * max_length, d, K, L, q_bf16 + (size_t)h * d, q_norm[h],
                           ind + (size_t)h * max_length, nnz[h], out_bf16 + (size_t)h * d,
                           max_value_expsum + h, max_value_expsum + H_total + h,
                           score ? score + (size_t)h * max_length : NULL);
    }
}

/* ------------------------------------------------------------------------------------------
 * Plain softmax attention of one q-head over a contiguous window of `len` rows (the sink +
 * local + generated tokens the reference hands to FlashInfer, models/attnserver.py:281-296),
 * returning the fp32 output and the base-2 LSE (FlashInfer convention), and the LSE-weighted
 * merge of two partial states (flashinfer.merge_state, models/attnserver.py:308; math restated
 * in SURVEY.md 8(a) a11).  FlashInfer is third-party and absent from the reference repository
 * (install.sh:4, unpinned wheel): "merge/window parity unpinned" -- these two follow the
 * published definition only.
 * ------------------------------------------------------------------------------------------ */
void orc_window_attention_head(const uint16_t *key /* [len][d] */, const uint16_t *value, int d, int len,
                               const uint16_t *q_bf16, float *out_f32, float *lse2) {
    if (len <= 0) {
        for (int i = 0; i < d; ++i) out_f32[i] = 0.f;
        *lse2 = -INFINITY;
        return;
    }
    double *s = (double *)malloc(sizeof(double) * (size_t)len);
    const double scale = 1.0 / sqrt((double)d);
    double m = -INFINITY;
    for (int j = 0; j < len; ++j) {
        double acc = 0.0;
        for (int i = 0; i < d; ++i) acc += (double)bf16_to_f32(q_bf16[i]) * (double)bf16_to_f32(key[(size_t)j * d + i]);
        s[j] = acc * scale;
        if (s[j] > m) m = s[j];
    }
    double sum = 0.0;
    for (int j = 0; j < len; ++j) {
        s[j] = exp(s[j] - m);
        sum += s[j];
    }
    for (int i = 0; i < d; ++i) {
        double acc = 0.0;
        for (int j = 0; j < len; ++j) acc += s[j] * (double)bf16_to_f32(value[(size_t)j * d + i]);
        out_f32[i] = (float)(acc / sum);
    }
    *lse2 = (float)(log2(sum) + m * M_LOG2E);
    free(s);
}

void orc_merge_state(const float *o_a, float lse2_a, const float *o_b, float lse2_b, int d, float *o, float *lse2) {
    float m = lse2_a > lse2_b ? lse2_a : lse2_b;
    if (m == -INFINITY) {
        for (int i = 0; i < d; ++i) o[i] = 0.f;
        *lse2 = -INFINITY;
        return;
    }
    double wa = exp2((double)lse2_a - m), wb = exp2((double)lse2_b - m);
    for (int i = 0; i < d; ++i) o[i] = (float)((o_a[i] * wa + o_b[i] * wb) / (wa + wb));
    *lse2 = (float)(m + log2(wa + wb));
}
