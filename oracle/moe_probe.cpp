// oracle/moe_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_ARGSORT and GGML_OP_SUM_ROWS graphs (the router ops of a mixture-of-experts FFN) on a named device, through the
// UNMODIFIED reference's public API (ggml_argsort / ggml_sum_rows, ggml_backend_*), built into oracle/_ref/libggml_moe_probe.so and driven
// from Python with ctypes (oracle/moe.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with
// probe_load_backend of libggml_probe.so) it is this repository's kernel.  Nothing here is on the product path.

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

namespace {

// the f32 source of shape ne, read through a view of a larger parent when view != 0:
//   view 1: every row padded by 3 floats (parent [ne0 + 3, ne1, ne2, ne3]): strided, evenly spaced rows
//   view 2: the corner of a parent [ne0 * 2, ne1 * 2, ne2 * 3, ne3] (what test-backend-ops does with v = 1): rows not evenly spaced
ggml_tensor * source(ggml_context * ctx, const int64_t * ne, int view, ggml_tensor ** parent) {
    if (view == 1) *parent = ggml_new_tensor_4d(ctx, GGML_TYPE_F32, ne[0] + 3, ne[1], ne[2], ne[3]);
    else if (view == 2) *parent = ggml_new_tensor_4d(ctx, GGML_TYPE_F32, ne[0] * 2, ne[1] * 2, ne[2] * 3, ne[3]);
    else return *parent = ggml_new_tensor_4d(ctx, GGML_TYPE_F32, ne[0], ne[1], ne[2], ne[3]);
    const ggml_tensor * p = *parent;
    return ggml_view_4d(ctx, *parent, ne[0], ne[1], ne[2], ne[3], p->nb[1], p->nb[2], p->nb[3], 0);
}

// build the one-node graph of `r` and run it on `dev`; x fills the parent, out receives r (contiguous)
int run(const char * dev, ggml_context * ctx, ggml_tensor * parent, ggml_tensor * r, const float * x, void * out) {
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
        ggml_backend_tensor_set(parent, x, 0, ggml_nbytes(parent));
        ggml_backend_graph_compute(be, gf);
        ggml_backend_tensor_get(r, out, 0, ggml_nbytes(r));
    }
    if (buf) ggml_backend_buffer_free(buf);
    ggml_free(ctx);
    ggml_backend_free(be);
    return rc;
}

ggml_context * new_ctx() {
    ggml_init_params ip = { ggml_tensor_overhead() * 8 + ggml_graph_overhead(), nullptr, true };
    return ggml_init(ip);
}

} // namespace

extern "C" {

// out (i32, ne0*ne1*ne2*ne3) = ARGSORT(x, order) on device `dev`; x holds the parent tensor (see source()).
// Returns 0, -1 (no such device), -2 (the device declines the node), -3 (allocation failed).
int probe_argsort(const char * dev, const int64_t * ne, int view, int order, const float * x, int32_t * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * parent;
    ggml_tensor * a = source(ctx, ne, view, &parent);
    return run(dev, ctx, parent, ggml_argsort(ctx, a, (ggml_sort_order) order), x, out);
}

// out (f32, ne1*ne2*ne3) = SUM_ROWS(x) on device `dev`; as probe_argsort
int probe_sum_rows(const char * dev, const int64_t * ne, int view, const float * x, float * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * parent;
    ggml_tensor * a = source(ctx, ne, view, &parent);
    return run(dev, ctx, parent, ggml_sum_rows(ctx, a), x, out);
}

} // extern "C"
