// oracle/ssm_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_CONCAT, GGML_OP_SSM_CONV and GGML_OP_SSM_SCAN graphs (the ops of a Mamba-1 layer) on a named device, through the
// UNMODIFIED reference's public API (ggml_concat / ggml_ssm_conv / ggml_ssm_scan, ggml_backend_*), built into oracle/_ref/libggml_ssm_probe.so
// and driven from Python with ctypes (oracle/ssm.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with
// probe_load_backend of libggml_probe.so) it is this repository's kernel.  Sources can be strided and transposed views, as in the Mamba
// graph.  Nothing here is on the product path.

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

#include <vector>

namespace {

// a source of shape ne read through a view of its own parent tensor (oracle/ssm.py mirrors the parent shapes):
//   view 0: contiguous (the parent itself)
//   view 1: the corner of a parent [2 ne0, 4 ne1, 3 ne2, ne3] (test-backend-ops' non-contiguous CONCAT operand): strided rows and planes
//   view 2: the transpose of a contiguous parent [ne1, ne0, ne2, ne3]: nb0 is a row stride (TRANSPOSE(x) in the Mamba layer)
//   view 3: rows packed, planes spread: the corner of a parent [ne0, ne1 + 3, ne2, ne3] (an SSM_CONV input with a free nb2)
ggml_tensor * source(ggml_context * ctx, ggml_type type, const int64_t * ne, int view, std::vector<ggml_tensor *> & parents) {
    ggml_tensor * p;
    switch (view) {
        case 1: p = ggml_new_tensor_4d(ctx, type, ne[0] * 2, ne[1] * 4, ne[2] * 3, ne[3]); break;
        case 2: p = ggml_new_tensor_4d(ctx, type, ne[1], ne[0], ne[2], ne[3]); break;
        case 3: p = ggml_new_tensor_4d(ctx, type, ne[0], ne[1] + 3, ne[2], ne[3]); break;
        default: p = ggml_new_tensor_4d(ctx, type, ne[0], ne[1], ne[2], ne[3]); break;
    }
    parents.push_back(p);
    if (view == 1 || view == 3) return ggml_view_4d(ctx, p, ne[0], ne[1], ne[2], ne[3], p->nb[1], p->nb[2], p->nb[3], 0);
    if (view == 2) return ggml_transpose(ctx, p);
    return p;
}

// build the one-node graph of `r` and run it on `dev`; data[i] fills parents[i], out receives r (contiguous)
int run(const char * dev, ggml_context * ctx, const std::vector<ggml_tensor *> & parents, const void * const * data, ggml_tensor * r, void * out) {
    ggml_backend_dev_t d = ggml_backend_dev_by_name(dev);
    ggml_backend_t be = d ? ggml_backend_dev_init(d, nullptr) : nullptr;
    if (!be) { ggml_free(ctx); return -1; }
    if (ggml_backend_is_cpu(be)) ggml_backend_cpu_set_n_threads(be, 4);
    ggml_cgraph * gf = ggml_new_graph(ctx);
    ggml_build_forward_expand(gf, r);
    int rc = 0;
    ggml_backend_buffer_t buf = nullptr;
    if (!ggml_backend_supports_op(be, r)) rc = -2;
    else if (!(buf = ggml_backend_alloc_ctx_tensors(ctx, be))) rc = -3;
    else {
        for (size_t i = 0; i < parents.size(); ++i) ggml_backend_tensor_set(parents[i], data[i], 0, ggml_nbytes(parents[i]));
        ggml_backend_graph_compute(be, gf);
        ggml_backend_tensor_get(r, out, 0, ggml_nbytes(r));
    }
    if (buf) ggml_backend_buffer_free(buf);
    ggml_free(ctx);
    ggml_backend_free(be);
    return rc;
}

ggml_context * new_ctx() {
    ggml_init_params ip = { ggml_tensor_overhead() * 24 + ggml_graph_overhead(), nullptr, true };
    return ggml_init(ip);
}

} // namespace

extern "C" {

// out (ne of the result, contiguous) = CONCAT(a, b, dim) on device `dev`; a has shape ne_a, b shape ne_b, each read through its view
// (see source()); type 0 f32, 1 i32, 2 f16.  data: the two parents' bytes.
// Returns 0, -1 (no such device), -2 (the device declines the node), -3 (allocation failed).
int probe_concat(const char * dev, int type, const int64_t * ne_a, int view_a, const int64_t * ne_b, int view_b, int dim, const void * const * data, void * out) {
    ggml_context * ctx = new_ctx();
    std::vector<ggml_tensor *> parents;
    const ggml_type t = type == 1 ? GGML_TYPE_I32 : type == 2 ? GGML_TYPE_F16 : GGML_TYPE_F32;
    ggml_tensor * a = source(ctx, t, ne_a, view_a, parents);
    ggml_tensor * b = source(ctx, t, ne_b, view_b, parents);
    return run(dev, ctx, parents, data, ggml_concat(ctx, a, b, dim), out);
}

// out f32 [d_inner, n_t, n_s] = SSM_CONV(sx, c): sx [d_conv - 1 + n_t, d_inner, n_s] through view_sx (0 or 3; 1 gives rows that are not
// packed, which ggml-cpu asserts against: only for asking a device whether it declines), c [d_conv, d_inner] through view_c (0 or 3;
// 1 gives a row stride ggml-cpu does not honour: it reads row i1 at i1 * d_conv)
int probe_ssm_conv(const char * dev, int64_t d_conv, int64_t d_inner, int64_t n_t, int64_t n_s, int view_sx, int view_c, const void * const * data, float * out) {
    ggml_context * ctx = new_ctx();
    std::vector<ggml_tensor *> parents;
    const int64_t ne_sx[4] = { d_conv - 1 + n_t, d_inner, n_s, 1 }, ne_c[4] = { d_conv, d_inner, 1, 1 };
    ggml_tensor * sx = source(ctx, GGML_TYPE_F32, ne_sx, view_sx, parents);
    ggml_tensor * c = source(ctx, GGML_TYPE_F32, ne_c, view_c, parents);
    return run(dev, ctx, parents, data, ggml_ssm_conv(ctx, sx, c), out);
}

// out f32 (d_inner n_t n_s + d_state d_inner n_s: y, then the final states) = SSM_SCAN(s, x, dt, A, B, C).  s, x, dt, A are contiguous;
// bc_rank < 0: B and C are contiguous tensors of their own (data: s, x, dt, A, B, C); bc_rank >= 0: B and C are views of one
// x_db [bc_rank + 2 d_state, n_t, n_s] at element offsets bc_rank and bc_rank + d_state, as in the Mamba layer (data: s, x, dt, A, x_db)
int probe_ssm_scan(const char * dev, int64_t d_state, int64_t d_inner, int64_t n_t, int64_t n_s, int64_t bc_rank, const void * const * data, float * out) {
    ggml_context * ctx = new_ctx();
    std::vector<ggml_tensor *> parents;
    ggml_tensor * s = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, d_state, d_inner, n_s);
    ggml_tensor * x = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, d_inner, n_t, n_s);
    ggml_tensor * dt = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, d_inner, n_t, n_s);
    ggml_tensor * A = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, d_state, d_inner);
    parents = { s, x, dt, A };
    ggml_tensor * B, * C;
    if (bc_rank < 0) {
        B = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, d_state, n_t, n_s);
        C = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, d_state, n_t, n_s);
        parents.push_back(B);
        parents.push_back(C);
    } else {
        ggml_tensor * xdb = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, bc_rank + 2 * d_state, n_t, n_s);
        parents.push_back(xdb);
        B = ggml_view_3d(ctx, xdb, d_state, n_t, n_s, xdb->nb[1], xdb->nb[2], ggml_element_size(xdb) * bc_rank);
        C = ggml_view_3d(ctx, xdb, d_state, n_t, n_s, xdb->nb[1], xdb->nb[2], ggml_element_size(xdb) * (bc_rank + d_state));
    }
    return run(dev, ctx, parents, data, ggml_ssm_scan(ctx, s, x, dt, A, B, C), out);
}

} // extern "C"
