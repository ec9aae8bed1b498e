// oracle/pool_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_POOL_2D, GGML_OP_UPSCALE, GGML_OP_LEAKY_RELU and GGML_OP_REPEAT graphs on a named device, through the UNMODIFIED
// reference's public API (ggml_pool_2d / ggml_upscale_ext / ggml_leaky_relu / ggml_repeat, ggml_backend_*), built into
// oracle/_ref/libggml_pool_probe.so and driven from Python with ctypes (oracle/pool.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the
// plug-in, loaded beforehand with probe_load_backend of libggml_probe.so) it is this repository's kernel.  Nothing here is on the product path.

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

#include <vector>

namespace {

// The source of every probe, read through a view of its own parent.  spec (int64): type, the parent's ne[4], the view's ne[4], its
// nb1, nb2, nb3 (bytes), its byte offset, and 1 to read the view transposed (dims 0 and 1 swapped, ggml_transpose)
ggml_tensor * source(ggml_context * ctx, const int64_t * spec, ggml_tensor ** parent) {
    ggml_tensor * p = ggml_new_tensor(ctx, (ggml_type) spec[0], 4, spec + 1);
    *parent = p;
    ggml_tensor * v = ggml_view_4d(ctx, p, spec[5], spec[6], spec[7], spec[8], (size_t) spec[9], (size_t) spec[10], (size_t) spec[11], (size_t) spec[12]);
    return spec[13] ? ggml_transpose(ctx, v) : v;
}

// build the graph of `r` and run it on `dev` (every node must be supported); data fills the parent, out receives r (its ggml_nbytes)
int run(const char * dev, ggml_context * ctx, ggml_tensor * parent, const void * data, ggml_tensor * r, void * out) {
    ggml_backend_dev_t d = ggml_backend_dev_by_name(dev);
    ggml_backend_t be = d ? ggml_backend_dev_init(d, nullptr) : nullptr;
    if (!be) { ggml_free(ctx); return -1; }
    if (ggml_backend_is_cpu(be)) ggml_backend_cpu_set_n_threads(be, 4);
    ggml_cgraph * gf = ggml_new_graph(ctx);
    ggml_build_forward_expand(gf, r);
    int rc = 0;
    for (int i = 0; i < ggml_graph_n_nodes(gf); ++i) {
        ggml_tensor * n = ggml_graph_node(gf, i);
        if (n->op != GGML_OP_RESHAPE && n->op != GGML_OP_VIEW && n->op != GGML_OP_TRANSPOSE && !ggml_backend_supports_op(be, n)) rc = -2;
    }
    ggml_backend_buffer_t buf = nullptr;
    if (rc == 0 && !(buf = ggml_backend_alloc_ctx_tensors(ctx, be))) rc = -3;
    if (rc == 0) {
        ggml_backend_tensor_set(parent, data, 0, ggml_nbytes(parent));
        if (ggml_backend_graph_compute(be, gf) != GGML_STATUS_SUCCESS) rc = -4;
        else ggml_backend_tensor_get(r, out, 0, ggml_nbytes(r));
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

} // namespace

extern "C" {

// Every probe returns 0, -1 (no such device), -2 (the device declines a node), -3 (allocation failed) or -4 (compute failed).

// out (f32, packed [OW, OH, C, N]) = ggml_pool_2d(source, op, k0, k1, s0, s1, p0, p1) with ggml_pool_2d's float paddings
int probe_pool_2d(const char * dev, const int64_t * spec, int op, int k0, int k1, int s0, int s1, float p0, float p1, const void * data, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = source(ctx, spec, &parent);
    return run(dev, ctx, parent, data, ggml_pool_2d(ctx, x, (ggml_op_pool) op, k0, k1, s0, s1, p0, p1), out);
}

// out (f32, packed ne) = ggml_upscale_ext(source, ne)
int probe_upscale(const char * dev, const int64_t * spec, const int64_t * ne, const void * data, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = source(ctx, spec, &parent);
    return run(dev, ctx, parent, data, ggml_upscale_ext(ctx, x, (int) ne[0], (int) ne[1], (int) ne[2], (int) ne[3]), out);
}

// out = ggml_leaky_relu(source, slope, inplace); in place the result is the source view itself, so out receives ggml_nbytes of it (a
// packed source gives the packed result)
int probe_leaky_relu(const char * dev, const int64_t * spec, float slope, int inplace, const void * data, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = source(ctx, spec, &parent);
    return run(dev, ctx, parent, data, ggml_leaky_relu(ctx, x, slope, inplace != 0), out);
}

// out (the source's type, packed ne) = ggml_repeat(source, a tensor of shape ne)
int probe_repeat(const char * dev, const int64_t * spec, const int64_t * ne, const void * data, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = source(ctx, spec, &parent);
    ggml_tensor * shape = ggml_new_tensor(ctx, x->type, 4, ne);
    return run(dev, ctx, parent, data, ggml_repeat(ctx, x, shape), out);
}

} // extern "C"
