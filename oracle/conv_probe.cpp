// oracle/conv_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_IM2COL and GGML_OP_MUL_MAT (f16 x f16) graphs, and the two-node ggml_conv_1d that chains them, on a named device,
// through the UNMODIFIED reference's public API (ggml_im2col / ggml_mul_mat / ggml_conv_1d, ggml_backend_*), built into
// oracle/_ref/libggml_conv_probe.so and driven from Python with ctypes (oracle/conv.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the
// plug-in, loaded beforehand with probe_load_backend of libggml_probe.so) it is this repository's kernel.  Nothing here is on the product path.

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

#include <vector>

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

// build the graph of `r` and run it on `dev` (every node must be supported); data[i] fills parents[i], out receives r (contiguous)
int run(const char * dev, ggml_context * ctx, const std::vector<ggml_tensor *> & parents, const void * const * data, ggml_tensor * r, void * out) {
    ggml_backend_dev_t d = ggml_backend_dev_by_name(dev);
    ggml_backend_t be = d ? ggml_backend_dev_init(d, nullptr) : nullptr;
    if (!be) { ggml_free(ctx); return -1; }
    if (ggml_backend_is_cpu(be)) ggml_backend_cpu_set_n_threads(be, 4);
    ggml_cgraph * gf = ggml_new_graph(ctx);
    ggml_build_forward_expand(gf, r);
    int rc = 0;
    for (int i = 0; i < ggml_graph_n_nodes(gf); ++i) {
        ggml_tensor * n = ggml_graph_node(gf, i);
        if (n->op != GGML_OP_RESHAPE && n->op != GGML_OP_VIEW && !ggml_backend_supports_op(be, n)) rc = -2;
    }
    ggml_backend_buffer_t buf = nullptr;
    if (rc == 0 && !(buf = ggml_backend_alloc_ctx_tensors(ctx, be))) rc = -3;
    if (rc == 0) {
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

// out (dst, contiguous) = IM2COL(kernel, input) on device `dev`: kernel of type kernel_type (0 f32, 1 f16; only its extents are read)
// and shape ne_kernel, input f32 of shape ne_input through `view` (see input()), params = { s0, s1, p0, p1, d0, d1, is_2D }, dst of type
// dst_type (0 f32, 1 f16).  data: the input parent's bytes.  Returns 0, -1 (no such device), -2 (the device declines the node),
// -3 (allocation failed).
int probe_im2col(const char * dev, int kernel_type, const int64_t * ne_kernel, const int64_t * ne_input, int view, const int32_t * params, int dst_type,
                 const void * const * data, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * k = ggml_new_tensor(ctx, kernel_type ? GGML_TYPE_F16 : GGML_TYPE_F32, 4, ne_kernel);
    ggml_tensor * parent;
    ggml_tensor * x = input(ctx, ne_input, view, &parent);
    ggml_tensor * r = ggml_im2col(ctx, k, x, params[0], params[1], params[2], params[3], params[4], params[5], params[6] == 1,
                                  dst_type ? GGML_TYPE_F16 : GGML_TYPE_F32);
    return run(dev, ctx, { parent }, data, r, out);
}

// out f32 [N, M] = MUL_MAT(a, b): a f16 [K, M], b f16 [K, N]; b_view 0: packed, 1: rows padded to K + 8 elements (nb1 a multiple of 16
// bytes when K is a multiple of 8), 2: rows padded to K + 3 elements (nb1 not a multiple of 16 bytes).  ggml-cpu asserts nb0 == 2 for b.
// data: a's bytes, then b's parent's.
int probe_mul_mat_f16(const char * dev, int64_t M, int64_t N, int64_t K, int b_view, const void * const * data, float * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * a = ggml_new_tensor_2d(ctx, GGML_TYPE_F16, K, M);
    ggml_tensor * bp, * b;
    if (b_view == 1 || b_view == 2) { bp = ggml_new_tensor_2d(ctx, GGML_TYPE_F16, K + (b_view == 1 ? 8 : 3), N); b = ggml_view_2d(ctx, bp, K, N, bp->nb[1], 0); }
    else                            { bp = ggml_new_tensor_2d(ctx, GGML_TYPE_F16, K, N); b = bp; }
    return run(dev, ctx, { a, bp }, data, ggml_mul_mat(ctx, a, b), out);
}

// out f32 [OC, OL] (ggml: [OL, OC]) = ggml_conv_1d(kernel, x, s, p, d): kernel f16 [KW, IC, OC], x f32 [L, IC] -> IM2COL (f16) + MUL_MAT.
// data: the kernel's bytes, then x's.
int probe_conv_1d(const char * dev, int64_t KW, int64_t IC, int64_t OC, int64_t L, int s, int p, int d, const void * const * data, float * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * k = ggml_new_tensor_3d(ctx, GGML_TYPE_F16, KW, IC, OC);
    ggml_tensor * x = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, L, IC);
    return run(dev, ctx, { k, x }, data, ggml_conv_1d(ctx, k, x, s, p, d), out);
}

} // extern "C"
