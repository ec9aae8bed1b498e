// oracle/wkv_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_RWKV_WKV6, GGML_OP_GATED_LINEAR_ATTN, GGML_OP_SQR and GGML_OP_SQRT graphs (the ops of an RWKV-6 layer the plug-in once
// declined) on a named device, through the UNMODIFIED reference's public API (ggml_rwkv_wkv6 / ggml_gated_linear_attn / ggml_sqr /
// ggml_sqrt, ggml_backend_*), built into oracle/_ref/libggml_wkv_probe.so and driven from Python with ctypes (oracle/wkv.py).  On "CPU" it
// is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with probe_load_backend of libggml_probe.so) it is this repository's kernel.
// Nothing here is on the product path.

#include "probe_harness.h"

#include <algorithm>

namespace {

// k, v, a (r or q), b (td or g) f32 [S, H, T] and the state f32 [S S H, n_seqs], in the order the op takes them
void wkv_sources(ggml_context * ctx, int64_t S, int64_t H, int64_t T, int64_t n_seqs, ggml_tensor ** t) {
    for (int i = 0; i < 4; ++i) t[i] = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, S, H, T);
    t[4] = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, S * S * H, n_seqs);
}

// ggml-cpu's WKV6 / GLA return before an internal barrier on threads ith >= H, so the CPU runs them with at most H threads
int cpu_threads(int64_t H) { return (int) std::max<int64_t>(1, std::min<int64_t>(4, H)); }

} // namespace

extern "C" {

// Every probe returns probe_run's code (probe_harness.h).

// out f32 [S H, T + S n_seqs] (y, then the final states) = RWKV_WKV6(k, v, r, tf, td, state); data: k, v, r, tf [S, H], td, state.
// T need not be a multiple of n_seqs here (ggml_rwkv_wkv6 does not assert it): only for asking a device whether it declines.
int probe_rwkv_wkv6(const char * dev, int64_t S, int64_t H, int64_t T, int64_t n_seqs, const void * const * data, float * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * t[5];
    wkv_sources(ctx, S, H, T, n_seqs, t);
    ggml_tensor * tf = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, S, H);
    ggml_tensor * r = ggml_rwkv_wkv6(ctx, t[0], t[1], t[2], tf, t[3], t[4]);
    return probe_run(dev, ctx, r, { { t[0], data[0] }, { t[1], data[1] }, { t[2], data[2] }, { tf, data[3] }, { t[3], data[4] }, { t[4], data[5] } },
                     { { r, out } }, cpu_threads(H));
}

// out as above = GATED_LINEAR_ATTN(k, v, q, g, state, scale); data: k, v, q, g, state
int probe_gated_linear_attn(const char * dev, int64_t S, int64_t H, int64_t T, int64_t n_seqs, float scale, const void * const * data, float * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * t[5];
    wkv_sources(ctx, S, H, T, n_seqs, t);
    ggml_tensor * r = ggml_gated_linear_attn(ctx, t[0], t[1], t[2], t[3], t[4], scale);
    return probe_run(dev, ctx, r, { { t[0], data[0] }, { t[1], data[1] }, { t[2], data[2] }, { t[3], data[3] }, { t[4], data[4] } },
                     { { r, out } }, cpu_threads(H));
}

// out f32 [n] = SQR(x) (op 0) or SQRT(x) (op 1) of a contiguous f32 x [n]
int probe_sqr_sqrt(const char * dev, int op, int64_t n, const void * const * data, float * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * x = ggml_new_tensor_1d(ctx, GGML_TYPE_F32, n);
    ggml_tensor * r = op == 0 ? ggml_sqr(ctx, x) : ggml_sqrt(ctx, x);
    return probe_run(dev, ctx, r, { { x, data[0] } }, { { r, out } });
}

} // extern "C"
