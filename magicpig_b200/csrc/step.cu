// step.cu -- the lifecycle of a decode step: plan (lengths advance by T, the step's node records), then at most one rewind or
// accept per plan, and the host mirror of the lengths that the eager checks of the plans read; and the device-side reorder of
// requests that a beam-search step ends with (mpig_reorder_requests).
//
// Replaces attnserver.py:196-198 (plan(): kv_last_page_len += 1) and, beyond the reference, the verification steps of
// speculative decoding: chains of T tokens (mpig_plan_tokens / mpig_rewind) and token trees (mpig_plan_tree / mpig_accept).
#include <algorithm>

#include "common.cuh"

namespace mpig {

// mpig_rewind: both lengths of request b shrink by drop[b] in [0, T]; any other drop leaves the request untouched and raises bit 2
// of the context's error flags.  apply = 0: only the flag (an eager call that refuses changes no length).
__global__ void rewind_kernel(const int32_t *drop, int32_t *win_len, int32_t *dense_len, int32_t *err_flag, int B, int T, int apply) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B) {
        const int d = drop[b];
        if (d < 0 || d > T) {
            atomicOr(err_flag, 4);
            return;
        }
        if (!apply) return;
        win_len[b] = max(win_len[b] - d, 0);
        dense_len[b] = max(dense_len[b] - d, 0);
    }
}

// Lengths advance by T (1 for mpig_plan) and saturate at the capacity (the append then overwrites the last row); saturation of a
// store that is in use raises the context's device error flag (bit 0: sparse window = generation_buffer exhausted, bit 1: a dense
// cache reached its capacity: dcap = max_length, or min(dcap, dense_base[b] + tail_rows) with a base map in shared dense mode),
// readable with mpig_error_flags -- the host-side check in mpig_plan cannot see replays of a captured graph.
// The step's node records go to step_buf: the bases (lengths after the plan minus T), the parents and the ancestor masks (bit j of
// mask t: node j is node t or one of its ancestors).  parents == null: a chain (node t's parent is t - 1).  A malformed tree
// (parents[b][0] != -1 or parents[b][t] outside [0, t)) raises bit 3 and request b runs as a chain.  apply = 0: only that check
// (an eager mpig_plan_tree that refuses changes nothing).  A chunk step longer than TREE_MAX (mpig_plan_chunk) writes the bases
// only: its rows have no node records.
__global__ void plan_kernel(int32_t *win_len, int32_t *dense_len, int32_t *err_flag, int B, int T, int wcap, int dcap,
                            int has_window, int has_dense, int32_t *step_buf, const int32_t *parents, int apply,
                            const int32_t *dense_base, int tail_rows) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B) {
        const int TN = (T <= TREE_MAX) ? T : 0;   // nodes with records
        int par[TREE_MAX];
        bool ok = true;
        for (int t = 0; t < TN; ++t) {
            par[t] = parents ? parents[b * T + t] : t - 1;
            ok &= (t == 0) ? (par[t] == -1) : (par[t] >= 0 && par[t] < t);
        }
        if (!ok) {
            atomicOr(err_flag, 8);
            for (int t = 0; t < TN; ++t) par[t] = t - 1;
        }
        if (!apply) return;
        int w = win_len[b] + T, dl = dense_len[b] + T;
        if (dense_base) dcap = min(dcap, dense_base[b] + tail_rows);
        if (w > wcap) {
            w = wcap;
            if (has_window) atomicOr(err_flag, 1);
        }
        if (dl > dcap) {
            dl = dcap;
            if (has_dense) atomicOr(err_flag, 2);
        }
        win_len[b] = w;
        dense_len[b] = dl;
        int32_t *bases = step_bases(step_buf, B), *masks = step_masks(step_buf) + b * T, *pout = step_parents(step_buf, B) + b * T;
        bases[2 * b] = w - T;
        bases[2 * b + 1] = dl - T;
        uint32_t m[TREE_MAX];
        for (int t = 0; t < TN; ++t) {
            m[t] = (t > 0 ? m[par[t]] : 0u) | (1u << t);
            masks[t] = (int32_t)m[t];
            pout[t] = par[t];
        }
    }
}

// mpig_accept: per request b, the root path nodes[b][0..count[b]) of the pending step becomes the step's first count[b] rows.  One
// warp per (row-owning layer, request, kv-head); lane l moves 16-byte chunk l (+32, ...) of each record, and reads every chunk of
// the path before it writes any, so the in-place move needs no staging.  A path is valid when 0 <= count <= T, nodes[0] = 0 and
// parents[nodes[i]] = nodes[i-1]; an invalid one leaves request b untouched and raises bit 3.  Rows are addressed from the step
// bases plan_kernel recorded (never from the lengths this kernel rewrites) and stay inside each store's capacity; with a base map
// (shared dense mode) the dense entries are the request tails, where the step starts at row base - dense_base[b].  The warp of
// (table entry 0, b, kv-head 0) sets both lengths to base + count.  apply = 0: only the check.
__global__ void __launch_bounds__(256) accept_path_kernel(const AcceptLayer *layers, int n_layers, const int32_t *nodes,
                                                          const int32_t *count, const int32_t *step_buf, int32_t *win_len,
                                                          int32_t *dense_len, int32_t *err_flag, int B, int Hkv, int T, int rec16,
                                                          int apply, const int32_t *dense_base) {
    const int wid = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    const int nl = max(n_layers, 1);
    if (wid >= nl * B * Hkv) return;
    const int li = wid / (B * Hkv), b = (wid / Hkv) % B, head = wid % Hkv;
    const int32_t *par = step_parents(step_buf, B) + b * T;
    const int cnt = count[b];
    bool ok = cnt >= 0 && cnt <= T;
    int nd[TREE_MAX];
#pragma unroll
    for (int i = 0; i < TREE_MAX; ++i) {
        nd[i] = i;
        if (ok && i < cnt) {
            const int n = nodes[b * T + i];
            if (i == 0) ok = (n == 0);
            else ok = (n > 0 && n < T && par[n] == nd[i - 1]);
            nd[i] = n;
        }
    }
    const bool leader = (li == 0 && head == 0);
    if (!ok) {
        if (leader && lane == 0) atomicOr(err_flag, 8);
        return;
    }
    if (!apply) return;
    const int32_t *bases = step_bases(step_buf, B);
    if (li < n_layers) {
        const AcceptLayer ly = layers[li];
        const int base = bases[2 * b + ly.dense] - ((ly.dense && dense_base) ? dense_base[b] : 0);
        uint4 *rows = reinterpret_cast<uint4 *>(ly.rows + ((size_t)b * Hkv + head) * (size_t)ly.cap * rec16 * 16);
        for (int ch = lane; ch < rec16; ch += 32) {
            uint4 v[TREE_MAX];
#pragma unroll
            for (int i = 0; i < TREE_MAX; ++i) {
                const int src = base + nd[i];
                if (i < cnt && nd[i] != i && base + i >= 0 && src < ly.cap) v[i] = rows[(size_t)src * rec16 + ch];
            }
#pragma unroll
            for (int i = 0; i < TREE_MAX; ++i) {
                const int src = base + nd[i];
                if (i < cnt && nd[i] != i && base + i >= 0 && src < ly.cap) rows[(size_t)(base + i) * rec16 + ch] = v[i];
            }
        }
    }
    if (leader && lane == 0) {
        win_len[b] = max(bases[2 * b] + cnt, 0);
        dense_len[b] = max(bases[2 * b + 1] + cnt, 0);
    }
}

// mpig_reorder_requests: request b continues request s = src_of[b]'s sequence.  The map's rule -- 0 <= src_of[b] < B and
// src_of[src_of[b]] == src_of[b] -- is checked in full by every CTA before it writes anything; a bad map leaves every request
// untouched and raises bit 4.  The rule means no request the call reads from is written, so the copy runs in place, in one pass.
//   Rows b < B: one CTA per (table entry, kv-head, chunk of REORDER_ROWS rows) in column x (entry e owns columns
//   [x0_e, x0_e + Hkv * ceil(cap_e / REORDER_ROWS))); CTAs of a request that stays (s == b), or past s's rows, exit at once.  The
//   rows are s's window rows [0, win_len[s]), dense rows [0, dense_len[s]) or, with a base map (shared dense mode), tail rows
//   [0, dense_len[s] - dense_base[s]), each capped at the entry's capacity; chunk 0 of a sparse entry also copies s's avg_k.
//   The CTA of column 0 sets b's lengths and dense base to s's (one thread per request, as the accept kernel's leader), and
//   writes slot_of[s] into slot_stage[b] for every b: the host copies the staging into slot_of after the kernel, so that no
//   kernel writes the slot map (mpig_ctx::slot_of).
//   Row B (shared spill mode): every vis word is rewritten in a register by the one thread that owns it: bit b becomes bit
//   src_of[b] of the word's old value for every moved b (vis_rebind_kernel(src_of[b], b) for all of them at once).
// apply = 0: only the check (an eager call that refuses).
__global__ void __launch_bounds__(256) reorder_requests_kernel(const AcceptLayer *layers, int n_layers, const int32_t *src_of,
                                                               int32_t *win_len, int32_t *dense_len, int32_t *dense_base,
                                                               const int32_t *slot_of, int32_t *slot_stage, uint32_t *vis,
                                                               size_t vis_words, int32_t *err_flag, int B, int Hkv, int rec16,
                                                               int d16, int apply) {
    constexpr int T = 256, UN = REORDER_ROWS * 32 / T;
    const int tid = threadIdx.x, x = blockIdx.x, b = blockIdx.y;
    bool ok = true;
    for (int i = tid; i < B; i += T) {
        const int s = src_of[i];
        ok &= (s >= 0 && s < B) && src_of[s] == s;
    }
    ok = __syncthreads_and(ok);
    if (!ok) {
        if (x == 0 && b == 0 && tid == 0) atomicOr(err_flag, 16);
        if (x == 0 && b < B && tid == 0) slot_stage[b] = slot_of[b];   // the copy after the kernel leaves the map as it was
        return;
    }
    if (!apply) return;
    if (b == B) {   // the visibility map (B <= 32 in shared spill mode)
        __shared__ int s_src[32];
        if (tid < B) s_src[tid] = src_of[tid];
        __syncthreads();
        uint32_t moved = 0;
        for (int r = 0; r < B; ++r) moved |= (s_src[r] != r ? 1u : 0u) << r;
        for (size_t i = (size_t)x * T + tid; i < vis_words; i += (size_t)gridDim.x * T) {
            const uint32_t v = vis[i];
            uint32_t w = v & ~moved;
            for (uint32_t m = moved; m; m &= m - 1) {
                const int r = __ffs(m) - 1;
                w |= ((v >> s_src[r]) & 1u) << r;
            }
            vis[i] = w;
        }
        return;
    }
    const int s = src_of[b];
    if (x == 0 && tid == 0) {
        slot_stage[b] = slot_of[s];
        if (s != b) {
            win_len[b] = win_len[s];
            dense_len[b] = dense_len[s];
            if (dense_base) dense_base[b] = dense_base[s];
        }
    }
    if (s == b || n_layers == 0) return;
    __shared__ int s_entry;
    for (int e = tid; e < n_layers; e += T)
        if (layers[e].x0 <= x && (e + 1 == n_layers || layers[e + 1].x0 > x)) s_entry = e;
    __syncthreads();
    const AcceptLayer ly = layers[s_entry];
    const int nch = (ly.cap + REORDER_ROWS - 1) / REORDER_ROWS;
    const int head = (x - ly.x0) / nch, ch = (x - ly.x0) % nch;
    if (ly.avg_k && ch == 0 && tid < d16) {
        const uint4 *a = reinterpret_cast<const uint4 *>(ly.avg_k);
        reinterpret_cast<uint4 *>(ly.avg_k)[((size_t)b * Hkv + head) * d16 + tid] = a[((size_t)s * Hkv + head) * d16 + tid];
    }
    int n = ly.dense ? dense_len[s] - (dense_base ? dense_base[s] : 0) : win_len[s];
    n = min(max(n, 0), ly.cap);
    const int r0 = ch * REORDER_ROWS;
    if (r0 >= n) return;
    const int total = min(REORDER_ROWS, n - r0) * rec16;   // 16-byte chunks of the CTA's rows, contiguous in both requests
    const uint4 *src = reinterpret_cast<const uint4 *>(ly.rows) + (((size_t)s * Hkv + head) * ly.cap + r0) * rec16;
    uint4 *dst = reinterpret_cast<uint4 *>(ly.rows) + (((size_t)b * Hkv + head) * ly.cap + r0) * rec16;
    for (int c0 = 0; c0 < total; c0 += T * UN) {
        uint4 v[UN];
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const int i = c0 + u * T + tid;
            if (i < total) v[u] = src[i];
        }
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const int i = c0 + u * T + tid;
            if (i < total) dst[i] = v[u];
        }
    }
}

int read_lengths(const mpig_ctx *ctx, int b0, int n, int32_t *wl, int32_t *dl, cudaStream_t s) {
    if (wl) MPIG_CUDA(cudaMemcpyAsync(wl, ctx->win_len + b0, n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (dl) MPIG_CUDA(cudaMemcpyAsync(dl, ctx->dense_len + b0, n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    MPIG_CUDA(cudaStreamSynchronize(s));
    return MPIG_OK;
}

// the host-mirror checks of mpig_plan for a step of T tokens (nothing is modified when one fails)
static int plan_checks(mpig_ctx *ctx, int T, bool has_window, bool has_dense, const char *who) {
    for (int b = 0; b < ctx->cfg.batch_size; ++b) {
        MPIG_REQUIRE(!has_window || ctx->h_win_len[b] + T <= ctx->Wcap, MPIG_ESTATE,
                     "%s: request %d: the sparse window is full (%d rows = sink + local + generation_buffer); "
                     "raise generation_buffer or clear()", who, b, ctx->Wcap);
        MPIG_REQUIRE(!has_dense || ctx->h_dense_len[b] == 0 || ctx->h_dense_len[b] + T <= ctx->dense_cap(b), MPIG_ESTATE,
                     "%s: request %d: the dense KV cache is full (capacity %d rows: %s)", who, b, ctx->dense_cap(b),
                     ctx->dense_tail_rows > 0 ? "the prompt base + dense_tail_rows, or max_length" : "max_length");
    }
    return MPIG_OK;
}

// mpig_plan / mpig_plan_tokens / mpig_plan_tree: the host-mirror checks (exact until a plan is captured into a CUDA graph: replays
// advance only the device side), then every length advances by T on the device and the step's node records are written
static int plan_step(mpig_ctx *ctx, int T, cudaStream_t s, const char *who, const int32_t *parents = nullptr, bool chunk = false) {
    const int B = ctx->cfg.batch_size;
    int has_window = 0, has_dense = 0;
    for (const auto &ls : ctx->layers) {
        has_window |= (ls.sparse && ctx->Wcap > 0);
        has_dense |= (ls.dense && ls.dense_kv != nullptr);
    }
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    MPIG_CUDA(cudaStreamIsCapturing(s, &cap));
    if (cap != cudaStreamCaptureStatusNone) {
        ctx->h_len_exact = false;
        ctx->plan_captured = true;
    }
    if (ctx->h_len_exact) {
        const int rc = plan_checks(ctx, T, has_window, has_dense, who);
        if (rc) return rc;
        for (int b = 0; b < B; ++b) {
            ctx->h_win_len[b] = std::min(ctx->h_win_len[b] + T, ctx->Wcap);
            ctx->h_dense_len[b] = std::min(ctx->h_dense_len[b] + T, ctx->dense_cap(b));
        }
    }
    plan_kernel<<<(B + 127) / 128, 128, 0, s>>>(ctx->win_len, ctx->dense_len, ctx->err_flag, B, T, ctx->Wcap, ctx->cfg.max_length,
                                               has_window, has_dense, ctx->step_buf, parents, 1, ctx->dense_base_map(),
                                               ctx->dense_tail_rows);
    MPIG_LAUNCH_CHECK(ctx);
    ctx->pending.begin(T, parents != nullptr, chunk);
    return MPIG_OK;
}

// host restatement of the device checks (eager calls refuse before anything is modified)
static bool tree_ok(const int32_t *par, int T) {
    for (int t = 0; t < T; ++t)
        if ((t == 0) ? (par[t] != -1) : (par[t] < 0 || par[t] >= t)) return false;
    return true;
}
static bool path_ok(const int32_t *nodes, int cnt, const int32_t *par, int T) {
    if (cnt < 0 || cnt > T) return false;
    for (int i = 0; i < cnt; ++i) {
        const int n = nodes[i];
        if (i == 0 ? (n != 0) : (n <= 0 || n >= T || par[n] != nodes[i - 1])) return false;
    }
    return true;
}

static int launch_accept(mpig_ctx *ctx, const int32_t *nodes, const int32_t *count, int T, int apply, cudaStream_t s) {
    const int B = ctx->cfg.batch_size, Hkv = ctx->cfg.num_key_value_heads;
    const int warps = std::max(ctx->n_accept_layers, 1) * B * Hkv;
    accept_path_kernel<<<(warps + 7) / 8, 256, 0, s>>>((const AcceptLayer *)ctx->accept_layers, ctx->n_accept_layers, nodes, count,
                                                       ctx->step_buf, ctx->win_len, ctx->dense_len, ctx->err_flag, B, Hkv, T,
                                                       ctx->rec_bytes / 16, apply, ctx->dense_base_map());
    MPIG_LAUNCH_CHECK(ctx);
    return MPIG_OK;
}

// The calls whose device inputs a kernel checks (mpig_rewind, mpig_accept, the tree of mpig_plan_tree).  Under capture the inputs
// cannot be read at the call: launch(1) runs, and the kernel's own check leaves a bad request untouched and raises an error flag
// bit.  Eagerly, host_check(ok) copies the inputs to the host and judges them first, so that a refused call changes nothing and may
// be repeated: a bad input runs launch(0), which only raises the flag bit, and sets *refused.
template <class HostCheck, class Launch>
static int checked_launch(cudaStream_t s, bool *eager, bool *refused, HostCheck host_check, Launch launch) {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    MPIG_CUDA(cudaStreamIsCapturing(s, &cap));
    *eager = (cap == cudaStreamCaptureStatusNone);
    bool ok = true;
    if (*eager) {
        const int rc = host_check(ok);
        if (rc) return rc;
    }
    *refused = !ok;
    return launch(ok ? 1 : 0);
}

// apply = 1: the reorder kernel, then the new slot map from its staging into slot_of (a copy-engine call, a memcpy node under
// capture); apply = 0: one CTA that only raises the flag bit
static int launch_reorder(mpig_ctx *ctx, const int32_t *src_of, int apply, cudaStream_t s) {
    const int B = ctx->cfg.batch_size, Hkv = ctx->cfg.num_key_value_heads;
    const size_t words = ctx->shared_spill ? (size_t)ctx->C * ctx->cfg.max_length : 0;
    const dim3 grid(apply ? std::max(ctx->reorder_cols, 1) : 1, apply ? B + (words ? 1 : 0) : 1);
    reorder_requests_kernel<<<grid, 256, 0, s>>>((const AcceptLayer *)ctx->accept_layers, ctx->n_accept_layers, src_of, ctx->win_len,
                                                 ctx->dense_len, ctx->dense_base_map() ? ctx->dense_base : nullptr, ctx->slot_of,
                                                 ctx->slot_stage, ctx->vis, words, ctx->err_flag, B, Hkv, ctx->rec_bytes / 16,
                                                 ctx->cfg.head_dim / 8, apply);
    MPIG_LAUNCH_CHECK(ctx);
    if (apply) MPIG_CUDA(cudaMemcpyAsync(ctx->slot_of, ctx->slot_stage, B * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    return MPIG_OK;
}

// the host restatement of the reorder kernel's check
static bool reorder_map_ok(const int32_t *src_of, int B) {
    for (int b = 0; b < B; ++b) {
        const int s = src_of[b];
        if (s < 0 || s >= B || src_of[s] != s) return false;
    }
    return true;
}

// after an applied rewind / accept: the step ends, and the host mirror follows the device lengths (an eager call: they are the
// truth, so the eager checks of mpig_plan stay exact) or stops being exact (a captured one)
static int end_step(mpig_ctx *ctx, bool eager, cudaStream_t s) {
    ctx->pending.end();
    if (!eager) {
        ctx->h_len_exact = false;
        return MPIG_OK;
    }
    const int B = ctx->cfg.batch_size;
    std::vector<int32_t> wl(B), dl(B);
    const int rc = read_lengths(ctx, 0, B, wl.data(), dl.data(), s);
    if (rc) return rc;
    for (int b = 0; b < B; ++b) {
        ctx->h_win_len[b] = wl[b];
        ctx->h_dense_len[b] = dl[b];
    }
    return MPIG_OK;
}

}  // namespace mpig

using namespace mpig;

extern "C" {

int mpig_plan(mpig_ctx *ctx, void *stream) {
    mpig::DeviceGuard _dg(ctx);  // run on the context's device whatever the caller's current device is
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "mpig_plan: null context");
    return plan_step(ctx, 1, as_stream(stream), "mpig_plan");
}

int mpig_plan_tokens(mpig_ctx *ctx, int T, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "mpig_plan_tokens: null context");
    MPIG_REQUIRE(T >= 1 && T <= ctx->tok_max, MPIG_EINVAL,
                 "mpig_plan_tokens: T=%d outside [1, %d] (mpig_reserve_query_tokens sets the upper bound)", T, ctx->tok_max);
    return plan_step(ctx, T, as_stream(stream), "mpig_plan_tokens");
}

int mpig_plan_chunk(mpig_ctx *ctx, int T, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx, MPIG_EINVAL, "mpig_plan_chunk: null context");
    MPIG_REQUIRE(T >= 1 && T <= ctx->chunk_max, MPIG_EINVAL,
                 "mpig_plan_chunk: T=%d outside [1, %d] (mpig_reserve_chunk_tokens sets the upper bound)", T, ctx->chunk_max);
    return plan_step(ctx, T, as_stream(stream), "mpig_plan_chunk", nullptr, true);
}

int mpig_rewind(mpig_ctx *ctx, const int32_t *drop, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx && drop, MPIG_EINVAL, "mpig_rewind: null argument");
    MPIG_REQUIRE(ctx->pending.T > 0 && ctx->pending.open, MPIG_ESTATE,
                 "mpig_rewind: at most one rewind or accept per plan (no plan since the last one)");
    MPIG_REQUIRE(!ctx->pending.tree, MPIG_ESTATE, "mpig_rewind: the pending step is a tree (mpig_plan_tree); commit a path with mpig_accept");
    const int B = ctx->cfg.batch_size, T = ctx->pending.T;
    cudaStream_t s = as_stream(stream);
    bool eager = true, refused = false;
    const int rc = checked_launch(
        s, &eager, &refused,
        [&](bool &ok) -> int {
            std::vector<int32_t> dh(B);
            MPIG_CUDA(cudaMemcpyAsync(dh.data(), drop, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            MPIG_CUDA(cudaStreamSynchronize(s));
            for (int b = 0; b < B; ++b) ok &= (dh[b] >= 0 && dh[b] <= T);
            return MPIG_OK;
        },
        [&](int apply) -> int {
            rewind_kernel<<<(B + 127) / 128, 128, 0, s>>>(drop, ctx->win_len, ctx->dense_len, ctx->err_flag, B, T, apply);
            MPIG_LAUNCH_CHECK(ctx);
            return MPIG_OK;
        });
    if (rc) return rc;
    MPIG_REQUIRE(!refused, MPIG_EINVAL, "mpig_rewind: a drop outside [0, %d]; nothing was changed (error flag bit 2)", T);
    return end_step(ctx, eager, s);
}

int mpig_plan_tree(mpig_ctx *ctx, int T, const int32_t *parents, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx && parents, MPIG_EINVAL, "mpig_plan_tree: null argument");
    MPIG_REQUIRE(T >= 1 && T <= ctx->tok_max, MPIG_EINVAL,
                 "mpig_plan_tree: T=%d outside [1, %d] (mpig_reserve_query_tokens sets the upper bound)", T, ctx->tok_max);
    const int B = ctx->cfg.batch_size;
    cudaStream_t s = as_stream(stream);
    bool eager = true, refused = false;
    const int rc = checked_launch(
        s, &eager, &refused,
        [&](bool &ok) -> int {
            std::vector<int32_t> ph((size_t)B * T);
            MPIG_CUDA(cudaMemcpyAsync(ph.data(), parents, ph.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            MPIG_CUDA(cudaStreamSynchronize(s));
            for (int b = 0; b < B; ++b) ok &= tree_ok(ph.data() + (size_t)b * T, T);
            return MPIG_OK;
        },
        [&](int apply) -> int {
            if (apply) return plan_step(ctx, T, s, "mpig_plan_tree", parents);
            plan_kernel<<<(B + 127) / 128, 128, 0, s>>>(ctx->win_len, ctx->dense_len, ctx->err_flag, B, T, ctx->Wcap,
                                                       ctx->cfg.max_length, 0, 0, ctx->step_buf, parents, 0, nullptr, 0);
            MPIG_LAUNCH_CHECK(ctx);
            return MPIG_OK;
        });
    if (rc) return rc;
    MPIG_REQUIRE(!refused, MPIG_EINVAL,
                 "mpig_plan_tree: a malformed tree (parents[b][0] must be -1 and 0 <= parents[b][t] < t); nothing was changed "
                 "(error flag bit 3)");
    return MPIG_OK;
}

int mpig_accept(mpig_ctx *ctx, const int32_t *nodes, const int32_t *count, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx && nodes && count, MPIG_EINVAL, "mpig_accept: null argument");
    MPIG_REQUIRE(ctx->pending.T > 0 && ctx->pending.open, MPIG_ESTATE,
                 "mpig_accept: at most one rewind or accept per plan (no plan since the last one)");
    MPIG_REQUIRE(!ctx->pending.chunk, MPIG_ESTATE, "mpig_accept: the pending step is a chunk step (mpig_plan_chunk); use mpig_rewind");
    const int B = ctx->cfg.batch_size, T = ctx->pending.T;
    cudaStream_t s = as_stream(stream);
    bool eager = true, refused = false;
    const int rc = checked_launch(
        s, &eager, &refused,
        [&](bool &ok) -> int {
            // the paths are checked against the step's parents
            std::vector<int32_t> nh((size_t)B * T), ch(B), ph((size_t)B * T);
            MPIG_CUDA(cudaMemcpyAsync(nh.data(), nodes, nh.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            MPIG_CUDA(cudaMemcpyAsync(ch.data(), count, ch.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            MPIG_CUDA(cudaMemcpyAsync(ph.data(), step_parents(ctx->step_buf, B), ph.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            MPIG_CUDA(cudaStreamSynchronize(s));
            for (int b = 0; b < B; ++b) ok &= path_ok(nh.data() + (size_t)b * T, ch[b], ph.data() + (size_t)b * T, T);
            return MPIG_OK;
        },
        [&](int apply) { return launch_accept(ctx, nodes, count, T, apply, s); });
    if (rc) return rc;
    MPIG_REQUIRE(!refused, MPIG_EINVAL,
                 "mpig_accept: a path that is not a root path of the pending step (count outside [0, %d], nodes[0] != 0 or "
                 "parents[nodes[i]] != nodes[i-1]); nothing was changed (error flag bit 3)", T);
    return end_step(ctx, eager, s);
}

int mpig_reorder_requests(mpig_ctx *ctx, const int32_t *src_of, void *stream) {
    mpig::DeviceGuard _dg(ctx);
    MPIG_REQUIRE(ctx && src_of, MPIG_EINVAL, "mpig_reorder_requests: null argument");
    MPIG_REQUIRE(ctx->C < ctx->cfg.batch_size, MPIG_ESTATE,
                 "mpig_reorder_requests: every request owns its context slot (num_contexts = batch_size); create the context with "
                 "fewer slots to share one");
    const int B = ctx->cfg.batch_size;
    cudaStream_t s = as_stream(stream);
    bool eager = true, refused = false;
    std::vector<int32_t> sh(B);
    int rc = checked_launch(
        s, &eager, &refused,
        [&](bool &ok) -> int {
            MPIG_CUDA(cudaMemcpyAsync(sh.data(), src_of, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            MPIG_CUDA(cudaStreamSynchronize(s));
            ok = reorder_map_ok(sh.data(), B);
            return MPIG_OK;
        },
        [&](int apply) { return launch_reorder(ctx, src_of, apply, s); });
    if (rc) return rc;
    MPIG_REQUIRE(!refused, MPIG_EINVAL,
                 "mpig_reorder_requests: a map whose sources are not all fixed points (src_of[b] outside [0, %d) or "
                 "src_of[src_of[b]] != src_of[b]); nothing was changed (error flag bit 4)", B);
    if (!eager) {   // replays change the device maps only
        ctx->h_map_exact = false;
        ctx->reorder_captured = true;
    }
    rc = end_step(ctx, eager, s);   // the lengths' mirror, as after a rewind; the bases of the pending step are stale
    if (rc || !eager) return rc;
    if (!ctx->h_map_exact) return refresh_maps(ctx, s);
    std::vector<int> so = ctx->h_slot_of, db = ctx->h_dense_base;
    for (int b = 0; b < B; ++b) {
        ctx->h_slot_of[b] = so[sh[b]];
        ctx->h_dense_base[b] = db[sh[b]];
    }
    return MPIG_OK;
}

}  // extern "C"
