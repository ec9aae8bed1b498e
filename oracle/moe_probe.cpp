// oracle/moe_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_ARGSORT and GGML_OP_SUM_ROWS graphs (the router ops of a mixture-of-experts FFN) on a named device, through the
// UNMODIFIED reference's public API (ggml_argsort / ggml_sum_rows, ggml_backend_*), built into oracle/_ref/libggml_moe_probe.so and driven
// from Python with ctypes (oracle/moe.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with
// probe_load_backend of libggml_probe.so) it is this repository's kernel.  Nothing here is on the product path.

#include "probe_harness.h"

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

} // namespace

extern "C" {

// Every probe returns probe_run's code (probe_harness.h).

// out (i32, ne0*ne1*ne2*ne3) = ARGSORT(x, order) on device `dev`; x holds the parent tensor (see source())
int probe_argsort(const char * dev, const int64_t * ne, int view, int order, const float * x, int32_t * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * parent;
    ggml_tensor * r = ggml_argsort(ctx, source(ctx, ne, view, &parent), (ggml_sort_order) order);
    return probe_run(dev, ctx, r, { { parent, x } }, { { r, out } });
}

// out (f32, ne1*ne2*ne3) = SUM_ROWS(x) on device `dev`; as probe_argsort
int probe_sum_rows(const char * dev, const int64_t * ne, int view, const float * x, float * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * parent;
    ggml_tensor * r = ggml_sum_rows(ctx, source(ctx, ne, view, &parent));
    return probe_run(dev, ctx, r, { { parent, x } }, { { r, out } });
}

} // extern "C"
