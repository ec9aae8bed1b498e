// oracle/train_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_OUT_PROD, GGML_OP_CROSS_ENTROPY_LOSS, GGML_OP_CROSS_ENTROPY_LOSS_BACK, GGML_OP_OPT_STEP_ADAMW, GGML_OP_ARGMAX,
// GGML_OP_COUNT_EQUAL, GGML_OP_SUM, GGML_OP_REPEAT_BACK and STEP graphs on a named device, through the UNMODIFIED reference's public API
// (ggml_out_prod / ggml_cross_entropy_loss[_back] / ggml_opt_step_adamw / ggml_argmax / ggml_count_equal / ggml_sum / ggml_repeat_back /
// ggml_step, ggml_backend_*), built into oracle/_ref/libggml_train_probe.so and driven from Python with ctypes (oracle/train.py).  On "CPU"
// it is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with probe_load_backend of libggml_probe.so) it is this repository's
// kernel.  Nothing here is on the product path.

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

#include <vector>

namespace {

// A source read through a view of its own parent: the spec of oracle/pool.py's Source (type, parent ne[4], view ne[4], nb1..nb3, offset,
// transposed)
ggml_tensor * source(ggml_context * ctx, const int64_t * spec, ggml_tensor ** parent) {
    ggml_tensor * p = ggml_new_tensor(ctx, (ggml_type) spec[0], 4, spec + 1);
    *parent = p;
    ggml_tensor * v = ggml_view_4d(ctx, p, spec[5], spec[6], spec[7], spec[8], (size_t) spec[9], (size_t) spec[10], (size_t) spec[11], (size_t) spec[12]);
    return spec[13] ? ggml_transpose(ctx, v) : v;
}

ggml_context * new_ctx() {
    ggml_init_params ip = { ggml_tensor_overhead() * 24 + ggml_graph_overhead(), nullptr, true };
    return ggml_init(ip);
}

// build the graph of `r` and run it on `dev` (every node must be supported); data[i] fills parents[i]; outs[i] receives reads[i]
int run(const char * dev, ggml_context * ctx, const std::vector<ggml_tensor *> & parents, const std::vector<const void *> & data, ggml_tensor * r,
        const std::vector<ggml_tensor *> & reads, const std::vector<void *> & outs) {
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
        for (size_t i = 0; i < parents.size(); ++i) ggml_backend_tensor_set(parents[i], data[i], 0, ggml_nbytes(parents[i]));
        if (ggml_backend_graph_compute(be, gf) != GGML_STATUS_SUCCESS) rc = -4;
        else for (size_t i = 0; i < reads.size(); ++i) ggml_backend_tensor_get(reads[i], outs[i], 0, ggml_nbytes(reads[i]));
    }
    if (buf) ggml_backend_buffer_free(buf);
    ggml_free(ctx);
    ggml_backend_free(be);
    return rc;
}

ggml_tensor * packed(ggml_context * ctx, ggml_type t, const int64_t * ne) { return ggml_new_tensor(ctx, t, 4, ne); }

} // namespace

extern "C" {

// Every probe returns 0, -1 (no such device), -2 (the device declines a node), -3 (allocation failed) or -4 (compute failed).

// out (f32, packed) = ggml_out_prod(a, b) for two sources (specs as above)
int probe_out_prod(const char * dev, const int64_t * spec_a, const int64_t * spec_b, const void * a, const void * b, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * pa, * pb;
    ggml_tensor * ta = source(ctx, spec_a, &pa), * tb = source(ctx, spec_b, &pb);
    ggml_tensor * r = ggml_out_prod(ctx, ta, tb);
    return run(dev, ctx, { pa, pb }, { a, b }, r, { r }, { out });
}

// out (f32 [1]) = ggml_cross_entropy_loss(x, l), x and l packed of extents ne
int probe_cross_entropy_loss(const char * dev, const int64_t * ne, const void * x, const void * l, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * tx = packed(ctx, GGML_TYPE_F32, ne), * tl = packed(ctx, GGML_TYPE_F32, ne);
    ggml_tensor * r = ggml_cross_entropy_loss(ctx, tx, tl);
    return run(dev, ctx, { tx, tl }, { x, l }, r, { r }, { out });
}

// out (f32, packed) = ggml_cross_entropy_loss_back(grad [1], x, l)
int probe_cross_entropy_loss_back(const char * dev, const int64_t * ne, const void * grad, const void * x, const void * l, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * tg = ggml_new_tensor_1d(ctx, GGML_TYPE_F32, 1), * tx = packed(ctx, GGML_TYPE_F32, ne), * tl = packed(ctx, GGML_TYPE_F32, ne);
    ggml_tensor * r = ggml_cross_entropy_loss_back(ctx, tg, tx, tl);
    return run(dev, ctx, { tg, tx, tl }, { grad, x, l }, r, { r }, { out });
}

// one ggml_opt_step_adamw on w (packed, extents ne) with g, m, v and the 7 hyper-parameters; w, m, v are written back to out_w, out_m, out_v
int probe_opt_step_adamw(const char * dev, const int64_t * ne, const void * w, const void * g, const void * m, const void * v, const void * params,
                         void * out_w, void * out_m, void * out_v) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * tw = packed(ctx, GGML_TYPE_F32, ne), * tg = packed(ctx, GGML_TYPE_F32, ne), * tm = packed(ctx, GGML_TYPE_F32, ne),
                * tv = packed(ctx, GGML_TYPE_F32, ne), * tp = ggml_new_tensor_1d(ctx, GGML_TYPE_F32, 7);
    ggml_set_param(ctx, tw);
    ggml_tensor * r = ggml_opt_step_adamw(ctx, tw, tg, tm, tv, tp);
    return run(dev, ctx, { tw, tg, tm, tv, tp }, { w, g, m, v, params }, r, { tw, tm, tv }, { out_w, out_m, out_v });
}

// out (i32 [ne1]) = ggml_argmax(x), x f32 packed [ne0, ne1]
int probe_argmax(const char * dev, int64_t ne0, int64_t ne1, const void * x, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * tx = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, ne0, ne1);
    ggml_tensor * r = ggml_argmax(ctx, tx);
    return run(dev, ctx, { tx }, { x }, r, { r }, { out });
}

// out (i64 [1]) = ggml_count_equal(a, b), both i32 packed of extents ne
int probe_count_equal(const char * dev, const int64_t * ne, const void * a, const void * b, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * ta = packed(ctx, GGML_TYPE_I32, ne), * tb = packed(ctx, GGML_TYPE_I32, ne);
    ggml_tensor * r = ggml_count_equal(ctx, ta, tb);
    return run(dev, ctx, { ta, tb }, { a, b }, r, { r }, { out });
}

// out (f32 [1]) = ggml_sum(source)
int probe_sum(const char * dev, const int64_t * spec, const void * x, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * p;
    ggml_tensor * r = ggml_sum(ctx, source(ctx, spec, &p));
    return run(dev, ctx, { p }, { x }, r, { r }, { out });
}

// out (f32, packed [ne]) = ggml_repeat_back(source, a tensor of extents ne)
int probe_repeat_back(const char * dev, const int64_t * spec, const int64_t * ne, const void * x, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * p;
    ggml_tensor * src = source(ctx, spec, &p);
    ggml_tensor * r = ggml_repeat_back(ctx, src, packed(ctx, GGML_TYPE_F32, ne));
    return run(dev, ctx, { p }, { x }, r, { r }, { out });
}

// out (f32, packed) = ggml_step(x), x f32 packed of extents ne
int probe_step(const char * dev, const int64_t * ne, const void * x, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * tx = packed(ctx, GGML_TYPE_F32, ne);
    ggml_tensor * r = ggml_step(ctx, tx);
    return run(dev, ctx, { tx }, { x }, r, { r }, { out });
}

} // extern "C"
