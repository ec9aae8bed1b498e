// oracle/conv_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_IM2COL and GGML_OP_MUL_MAT (f16 x f16) graphs, and the two-node ggml_conv_1d that chains them, on a named device,
// through the UNMODIFIED reference's public API (ggml_im2col / ggml_mul_mat / ggml_conv_1d, ggml_backend_*), built into
// oracle/_ref/libggml_conv_probe.so and driven from Python with ctypes (oracle/conv.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the
// plug-in, loaded beforehand with probe_load_backend of libggml_probe.so) it is this repository's kernel.  Nothing here is on the product path.

#include "probe_harness.h"

namespace {

// the input of IM2COL, shape ne, read through a view of its own parent (oracle/conv.py mirrors the parent shapes):
//   view 0: contiguous (the parent itself)
//   view 1: rows packed, planes and images spread: the corner of a parent [ne0, ne1 + 3, ne2 + 2, ne3]
//   view 2: rows spread too: the corner of a parent [ne0 + 5, ne1 + 3, ne2 + 2, ne3] (ggml-cpu reads a channel's rows as packed
//           whatever nb1: the device must read the same elements)
ggml_tensor * input(ggml_context * ctx, const int64_t * ne, int view, ggml_tensor ** parent) {
    const int64_t pad0 = view == 2 ? 5 : 0, pad = view ? 1 : 0;
    ggml_tensor * p = ggml_new_tensor_4d(ctx, GGML_TYPE_F32, ne[0] + pad0, ne[1] + 3 * pad, ne[2] + 2 * pad, ne[3]);
    *parent = p;
    return view ? ggml_view_4d(ctx, p, ne[0], ne[1], ne[2], ne[3], p->nb[1], p->nb[2], p->nb[3], 0) : p;
}

} // namespace

extern "C" {

// Every probe returns probe_run's code (probe_harness.h).

// out (dst, contiguous) = IM2COL(kernel, input) on device `dev`: kernel of type kernel_type (0 f32, 1 f16; only its extents are read)
// and shape ne_kernel, input f32 of shape ne_input through `view` (see input()), params = { s0, s1, p0, p1, d0, d1, is_2D }, dst of type
// dst_type (0 f32, 1 f16).  data: the input parent's bytes.
int probe_im2col(const char * dev, int kernel_type, const int64_t * ne_kernel, const int64_t * ne_input, int view, const int32_t * params, int dst_type,
                 const void * const * data, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * k = ggml_new_tensor(ctx, kernel_type ? GGML_TYPE_F16 : GGML_TYPE_F32, 4, ne_kernel);
    ggml_tensor * parent;
    ggml_tensor * x = input(ctx, ne_input, view, &parent);
    ggml_tensor * r = ggml_im2col(ctx, k, x, params[0], params[1], params[2], params[3], params[4], params[5], params[6] == 1,
                                  dst_type ? GGML_TYPE_F16 : GGML_TYPE_F32);
    return probe_run(dev, ctx, r, { { parent, data[0] } }, { { r, out } });
}

// out f32 [N, M] = MUL_MAT(a, b): a f16 [K, M], b f16 [K, N]; b_view 0: packed, 1: rows padded to K + 8 elements (nb1 a multiple of 16
// bytes when K is a multiple of 8), 2: rows padded to K + 3 elements (nb1 not a multiple of 16 bytes).  ggml-cpu asserts nb0 == 2 for b.
// data: a's bytes, then b's parent's.
int probe_mul_mat_f16(const char * dev, int64_t M, int64_t N, int64_t K, int b_view, const void * const * data, float * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * a = ggml_new_tensor_2d(ctx, GGML_TYPE_F16, K, M);
    ggml_tensor * bp, * b;
    if (b_view == 1 || b_view == 2) { bp = ggml_new_tensor_2d(ctx, GGML_TYPE_F16, K + (b_view == 1 ? 8 : 3), N); b = ggml_view_2d(ctx, bp, K, N, bp->nb[1], 0); }
    else                            { bp = ggml_new_tensor_2d(ctx, GGML_TYPE_F16, K, N); b = bp; }
    ggml_tensor * r = ggml_mul_mat(ctx, a, b);
    return probe_run(dev, ctx, r, { { a, data[0] }, { bp, data[1] } }, { { r, out } });
}

// out f32 [OC, OL] (ggml: [OL, OC]) = ggml_conv_1d(kernel, x, s, p, d): kernel f16 [KW, IC, OC], x f32 [L, IC] -> IM2COL (f16) + MUL_MAT.
// data: the kernel's bytes, then x's.
int probe_conv_1d(const char * dev, int64_t KW, int64_t IC, int64_t OC, int64_t L, int s, int p, int d, const void * const * data, float * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * k = ggml_new_tensor_3d(ctx, GGML_TYPE_F16, KW, IC, OC);
    ggml_tensor * x = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, L, IC);
    ggml_tensor * r = ggml_conv_1d(ctx, k, x, s, p, d);
    return probe_run(dev, ctx, r, { { k, data[0] }, { x, data[1] } }, { { r, out } });
}

} // extern "C"
