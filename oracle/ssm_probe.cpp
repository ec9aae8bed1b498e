// oracle/ssm_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_CONCAT, GGML_OP_SSM_CONV and GGML_OP_SSM_SCAN graphs (the ops of a Mamba-1 layer) on a named device, through the
// UNMODIFIED reference's public API (ggml_concat / ggml_ssm_conv / ggml_ssm_scan, ggml_backend_*), built into oracle/_ref/libggml_ssm_probe.so
// and driven from Python with ctypes (oracle/ssm.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with
// probe_load_backend of libggml_probe.so) it is this repository's kernel.  Sources can be strided and transposed views, as in the Mamba
// graph.  Nothing here is on the product path.

#include "probe_harness.h"

namespace {

// a source of shape ne read through a view of its own parent tensor (oracle/ssm.py mirrors the parent shapes):
//   view 0: contiguous (the parent itself)
//   view 1: the corner of a parent [2 ne0, 4 ne1, 3 ne2, ne3] (test-backend-ops' non-contiguous CONCAT operand): strided rows and planes
//   view 2: the transpose of a contiguous parent [ne1, ne0, ne2, ne3]: nb0 is a row stride (TRANSPOSE(x) in the Mamba layer)
//   view 3: rows packed, planes spread: the corner of a parent [ne0, ne1 + 3, ne2, ne3] (an SSM_CONV input with a free nb2)
ggml_tensor * source(ggml_context * ctx, ggml_type type, const int64_t * ne, int view, ggml_tensor ** parent) {
    ggml_tensor * p;
    switch (view) {
        case 1: p = ggml_new_tensor_4d(ctx, type, ne[0] * 2, ne[1] * 4, ne[2] * 3, ne[3]); break;
        case 2: p = ggml_new_tensor_4d(ctx, type, ne[1], ne[0], ne[2], ne[3]); break;
        case 3: p = ggml_new_tensor_4d(ctx, type, ne[0], ne[1] + 3, ne[2], ne[3]); break;
        default: p = ggml_new_tensor_4d(ctx, type, ne[0], ne[1], ne[2], ne[3]); break;
    }
    *parent = p;
    if (view == 1 || view == 3) return ggml_view_4d(ctx, p, ne[0], ne[1], ne[2], ne[3], p->nb[1], p->nb[2], p->nb[3], 0);
    if (view == 2) return ggml_transpose(ctx, p);
    return p;
}

} // namespace

extern "C" {

// Every probe returns probe_run's code (probe_harness.h).

// out (ne of the result, contiguous) = CONCAT(a, b, dim) on device `dev`; a has shape ne_a, b shape ne_b, each read through its view
// (see source()); type 0 f32, 1 i32, 2 f16.  data: the two parents' bytes.
int probe_concat(const char * dev, int type, const int64_t * ne_a, int view_a, const int64_t * ne_b, int view_b, int dim, const void * const * data, void * out) {
    ggml_context * ctx = probe_ctx();
    const ggml_type t = type == 1 ? GGML_TYPE_I32 : type == 2 ? GGML_TYPE_F16 : GGML_TYPE_F32;
    ggml_tensor * pa, * pb;
    ggml_tensor * a = source(ctx, t, ne_a, view_a, &pa);
    ggml_tensor * b = source(ctx, t, ne_b, view_b, &pb);
    ggml_tensor * r = ggml_concat(ctx, a, b, dim);
    return probe_run(dev, ctx, r, { { pa, data[0] }, { pb, data[1] } }, { { r, out } });
}

// out f32 [d_inner, n_t, n_s] = SSM_CONV(sx, c): sx [d_conv - 1 + n_t, d_inner, n_s] through view_sx (0 or 3; 1 gives rows that are not
// packed, which ggml-cpu asserts against: only for asking a device whether it declines), c [d_conv, d_inner] through view_c (0 or 3;
// 1 gives a row stride ggml-cpu does not honour: it reads row i1 at i1 * d_conv)
int probe_ssm_conv(const char * dev, int64_t d_conv, int64_t d_inner, int64_t n_t, int64_t n_s, int view_sx, int view_c, const void * const * data, float * out) {
    ggml_context * ctx = probe_ctx();
    const int64_t ne_sx[4] = { d_conv - 1 + n_t, d_inner, n_s, 1 }, ne_c[4] = { d_conv, d_inner, 1, 1 };
    ggml_tensor * psx, * pc;
    ggml_tensor * sx = source(ctx, GGML_TYPE_F32, ne_sx, view_sx, &psx);
    ggml_tensor * c = source(ctx, GGML_TYPE_F32, ne_c, view_c, &pc);
    ggml_tensor * r = ggml_ssm_conv(ctx, sx, c);
    return probe_run(dev, ctx, r, { { psx, data[0] }, { pc, data[1] } }, { { r, out } });
}

// out f32 (d_inner n_t n_s + d_state d_inner n_s: y, then the final states) = SSM_SCAN(s, x, dt, A, B, C).  s, x, dt, A are contiguous;
// bc_rank < 0: B and C are contiguous tensors of their own (data: s, x, dt, A, B, C); bc_rank >= 0: B and C are views of one
// x_db [bc_rank + 2 d_state, n_t, n_s] at element offsets bc_rank and bc_rank + d_state, as in the Mamba layer (data: s, x, dt, A, x_db)
int probe_ssm_scan(const char * dev, int64_t d_state, int64_t d_inner, int64_t n_t, int64_t n_s, int64_t bc_rank, const void * const * data, float * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * s = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, d_state, d_inner, n_s);
    ggml_tensor * x = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, d_inner, n_t, n_s);
    ggml_tensor * dt = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, d_inner, n_t, n_s);
    ggml_tensor * A = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, d_state, d_inner);
    probe_uploads up = { { s, data[0] }, { x, data[1] }, { dt, data[2] }, { A, data[3] } };
    ggml_tensor * B, * C;
    if (bc_rank < 0) {
        B = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, d_state, n_t, n_s);
        C = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, d_state, n_t, n_s);
        up.push_back({ B, data[4] });
        up.push_back({ C, data[5] });
    } else {
        ggml_tensor * xdb = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, bc_rank + 2 * d_state, n_t, n_s);
        up.push_back({ xdb, data[4] });
        B = ggml_view_3d(ctx, xdb, d_state, n_t, n_s, xdb->nb[1], xdb->nb[2], ggml_element_size(xdb) * bc_rank);
        C = ggml_view_3d(ctx, xdb, d_state, n_t, n_s, xdb->nb[1], xdb->nb[2], ggml_element_size(xdb) * (bc_rank + d_state));
    }
    ggml_tensor * r = ggml_ssm_scan(ctx, s, x, dt, A, B, C);
    return probe_run(dev, ctx, r, up, { { r, out } });
}

} // extern "C"
