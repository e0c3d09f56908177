// step.cu -- the lifecycle of a decode step: plan (lengths advance by T, the step's node records), then at most one rewind or
// accept per plan, and the host mirror of the lengths that the eager checks of the plans read.
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
// (an eager mpig_plan_tree that refuses changes nothing).
__global__ void plan_kernel(int32_t *win_len, int32_t *dense_len, int32_t *err_flag, int B, int T, int wcap, int dcap,
                            int has_window, int has_dense, int32_t *step_buf, const int32_t *parents, int apply,
                            const int32_t *dense_base, int tail_rows) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B) {
        int par[TREE_MAX];
        bool ok = true;
        for (int t = 0; t < T; ++t) {
            par[t] = parents ? parents[b * T + t] : t - 1;
            ok &= (t == 0) ? (par[t] == -1) : (par[t] >= 0 && par[t] < t);
        }
        if (!ok) {
            atomicOr(err_flag, 8);
            for (int t = 0; t < T; ++t) par[t] = t - 1;
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
        for (int t = 0; t < T; ++t) {
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
static int plan_step(mpig_ctx *ctx, int T, cudaStream_t s, const char *who, const int32_t *parents = nullptr) {
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
    ctx->pending.begin(T, parents != nullptr);
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

}  // extern "C"
