// oracle/wkv_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_RWKV_WKV6, GGML_OP_GATED_LINEAR_ATTN, GGML_OP_SQR and GGML_OP_SQRT graphs (the ops of an RWKV-6 layer the plug-in once
// declined) on a named device, through the UNMODIFIED reference's public API (ggml_rwkv_wkv6 / ggml_gated_linear_attn / ggml_sqr /
// ggml_sqrt, ggml_backend_*), built into oracle/_ref/libggml_wkv_probe.so and driven from Python with ctypes (oracle/wkv.py).  On "CPU" it
// is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with probe_load_backend of libggml_probe.so) it is this repository's kernel.
// Nothing here is on the product path.

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

#include <algorithm>
#include <vector>

namespace {

// build the one-node graph of `r` and run it on `dev`; data[i] fills srcs[i], out receives r (contiguous).  ggml-cpu's WKV6 / GLA return
// before an internal barrier on threads ith >= H, so the CPU runs with at most `max_threads` threads (the head count for those two ops).
int run(const char * dev, ggml_context * ctx, const std::vector<ggml_tensor *> & srcs, const void * const * data, ggml_tensor * r, void * out,
        int max_threads) {
    ggml_backend_dev_t d = ggml_backend_dev_by_name(dev);
    ggml_backend_t be = d ? ggml_backend_dev_init(d, nullptr) : nullptr;
    if (!be) { ggml_free(ctx); return -1; }
    if (ggml_backend_is_cpu(be)) ggml_backend_cpu_set_n_threads(be, std::max(1, std::min(4, max_threads)));
    ggml_cgraph * gf = ggml_new_graph(ctx);
    ggml_build_forward_expand(gf, r);
    int rc = 0;
    ggml_backend_buffer_t buf = nullptr;
    if (!ggml_backend_supports_op(be, r)) rc = -2;
    else if (!(buf = ggml_backend_alloc_ctx_tensors(ctx, be))) rc = -3;
    else {
        for (size_t i = 0; i < srcs.size(); ++i) ggml_backend_tensor_set(srcs[i], data[i], 0, ggml_nbytes(srcs[i]));
        ggml_backend_graph_compute(be, gf);
        ggml_backend_tensor_get(r, out, 0, ggml_nbytes(r));
    }
    if (buf) ggml_backend_buffer_free(buf);
    ggml_free(ctx);
    ggml_backend_free(be);
    return rc;
}

ggml_context * new_ctx() {
    ggml_init_params ip = { ggml_tensor_overhead() * 16 + ggml_graph_overhead(), nullptr, true };
    return ggml_init(ip);
}

// k, v, a (r or q), b (td or g) f32 [S, H, T] and the state f32 [S S H, n_seqs], in the order the op takes them
void wkv_sources(ggml_context * ctx, int64_t S, int64_t H, int64_t T, int64_t n_seqs, std::vector<ggml_tensor *> & t) {
    for (int i = 0; i < 4; ++i) t.push_back(ggml_new_tensor_3d(ctx, GGML_TYPE_F32, S, H, T));
    t.push_back(ggml_new_tensor_2d(ctx, GGML_TYPE_F32, S * S * H, n_seqs));
}

} // namespace

extern "C" {

// out f32 [S H, T + S n_seqs] (y, then the final states) = RWKV_WKV6(k, v, r, tf, td, state); data: k, v, r, tf [S, H], td, state.
// T need not be a multiple of n_seqs here (ggml_rwkv_wkv6 does not assert it): only for asking a device whether it declines.
// Returns 0, -1 (no such device), -2 (the device declines the node), -3 (allocation failed).
int probe_rwkv_wkv6(const char * dev, int64_t S, int64_t H, int64_t T, int64_t n_seqs, const void * const * data, float * out) {
    ggml_context * ctx = new_ctx();
    std::vector<ggml_tensor *> t;
    wkv_sources(ctx, S, H, T, n_seqs, t);
    ggml_tensor * tf = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, S, H);
    const std::vector<ggml_tensor *> srcs = { t[0], t[1], t[2], tf, t[3], t[4] };
    return run(dev, ctx, srcs, data, ggml_rwkv_wkv6(ctx, t[0], t[1], t[2], tf, t[3], t[4]), out, (int) H);
}

// out as above = GATED_LINEAR_ATTN(k, v, q, g, state, scale); data: k, v, q, g, state
int probe_gated_linear_attn(const char * dev, int64_t S, int64_t H, int64_t T, int64_t n_seqs, float scale, const void * const * data, float * out) {
    ggml_context * ctx = new_ctx();
    std::vector<ggml_tensor *> t;
    wkv_sources(ctx, S, H, T, n_seqs, t);
    return run(dev, ctx, t, data, ggml_gated_linear_attn(ctx, t[0], t[1], t[2], t[3], t[4], scale), out, (int) H);
}

// out f32 [n] = SQR(x) (op 0) or SQRT(x) (op 1) of a contiguous f32 x [n]
int probe_sqr_sqrt(const char * dev, int op, int64_t n, const void * const * data, float * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * x = ggml_new_tensor_1d(ctx, GGML_TYPE_F32, n);
    return run(dev, ctx, { x }, data, op == 0 ? ggml_sqr(ctx, x) : ggml_sqrt(ctx, x), out, 4);
}

} // extern "C"
