// oracle/train_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_OUT_PROD, GGML_OP_CROSS_ENTROPY_LOSS, GGML_OP_CROSS_ENTROPY_LOSS_BACK, GGML_OP_OPT_STEP_ADAMW, GGML_OP_ARGMAX,
// GGML_OP_COUNT_EQUAL, GGML_OP_SUM, GGML_OP_REPEAT_BACK and STEP graphs on a named device, through the UNMODIFIED reference's public API
// (ggml_out_prod / ggml_cross_entropy_loss[_back] / ggml_opt_step_adamw / ggml_argmax / ggml_count_equal / ggml_sum / ggml_repeat_back /
// ggml_step, ggml_backend_*), built into oracle/_ref/libggml_train_probe.so and driven from Python with ctypes (oracle/train.py).  On "CPU"
// it is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with probe_load_backend of libggml_probe.so) it is this repository's
// kernel.  Nothing here is on the product path.

#include "probe_harness.h"

namespace {

ggml_tensor * packed(ggml_context * ctx, ggml_type t, const int64_t * ne) { return ggml_new_tensor(ctx, t, 4, ne); }

} // namespace

extern "C" {

// Every probe returns probe_run's code (probe_harness.h).

// out (f32, packed) = ggml_out_prod(a, b) for two sources (specs: probe_view_source's)
int probe_out_prod(const char * dev, const int64_t * spec_a, const int64_t * spec_b, const void * a, const void * b, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * pa, * pb;
    ggml_tensor * ta = probe_view_source(ctx, spec_a, &pa), * tb = probe_view_source(ctx, spec_b, &pb);
    ggml_tensor * r = ggml_out_prod(ctx, ta, tb);
    return probe_run(dev, ctx, r, { { pa, a }, { pb, b } }, { { r, out } });
}

// out (f32 [1]) = ggml_cross_entropy_loss(x, l), x and l packed of extents ne
int probe_cross_entropy_loss(const char * dev, const int64_t * ne, const void * x, const void * l, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * tx = packed(ctx, GGML_TYPE_F32, ne), * tl = packed(ctx, GGML_TYPE_F32, ne);
    ggml_tensor * r = ggml_cross_entropy_loss(ctx, tx, tl);
    return probe_run(dev, ctx, r, { { tx, x }, { tl, l } }, { { r, out } });
}

// out (f32, packed) = ggml_cross_entropy_loss_back(grad [1], x, l)
int probe_cross_entropy_loss_back(const char * dev, const int64_t * ne, const void * grad, const void * x, const void * l, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * tg = ggml_new_tensor_1d(ctx, GGML_TYPE_F32, 1), * tx = packed(ctx, GGML_TYPE_F32, ne), * tl = packed(ctx, GGML_TYPE_F32, ne);
    ggml_tensor * r = ggml_cross_entropy_loss_back(ctx, tg, tx, tl);
    return probe_run(dev, ctx, r, { { tg, grad }, { tx, x }, { tl, l } }, { { r, out } });
}

// one ggml_opt_step_adamw on w (packed, extents ne) with g, m, v and the 7 hyper-parameters; w, m, v are written back to out_w, out_m, out_v
int probe_opt_step_adamw(const char * dev, const int64_t * ne, const void * w, const void * g, const void * m, const void * v, const void * params,
                         void * out_w, void * out_m, void * out_v) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * tw = packed(ctx, GGML_TYPE_F32, ne), * tg = packed(ctx, GGML_TYPE_F32, ne), * tm = packed(ctx, GGML_TYPE_F32, ne),
                * tv = packed(ctx, GGML_TYPE_F32, ne), * tp = ggml_new_tensor_1d(ctx, GGML_TYPE_F32, 7);
    ggml_set_param(ctx, tw);
    ggml_tensor * r = ggml_opt_step_adamw(ctx, tw, tg, tm, tv, tp);
    return probe_run(dev, ctx, r, { { tw, w }, { tg, g }, { tm, m }, { tv, v }, { tp, params } },
                     { { tw, out_w }, { tm, out_m }, { tv, out_v } });
}

// out (i32 [ne1]) = ggml_argmax(x), x f32 packed [ne0, ne1]
int probe_argmax(const char * dev, int64_t ne0, int64_t ne1, const void * x, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * tx = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, ne0, ne1);
    ggml_tensor * r = ggml_argmax(ctx, tx);
    return probe_run(dev, ctx, r, { { tx, x } }, { { r, out } });
}

// out (i64 [1]) = ggml_count_equal(a, b), both i32 packed of extents ne
int probe_count_equal(const char * dev, const int64_t * ne, const void * a, const void * b, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * ta = packed(ctx, GGML_TYPE_I32, ne), * tb = packed(ctx, GGML_TYPE_I32, ne);
    ggml_tensor * r = ggml_count_equal(ctx, ta, tb);
    return probe_run(dev, ctx, r, { { ta, a }, { tb, b } }, { { r, out } });
}

// out (f32 [1]) = ggml_sum(source)
int probe_sum(const char * dev, const int64_t * spec, const void * x, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * p;
    ggml_tensor * r = ggml_sum(ctx, probe_view_source(ctx, spec, &p));
    return probe_run(dev, ctx, r, { { p, x } }, { { r, out } });
}

// out (f32, packed [ne]) = ggml_repeat_back(source, a tensor of extents ne)
int probe_repeat_back(const char * dev, const int64_t * spec, const int64_t * ne, const void * x, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * p;
    ggml_tensor * src = probe_view_source(ctx, spec, &p);
    ggml_tensor * r = ggml_repeat_back(ctx, src, packed(ctx, GGML_TYPE_F32, ne));
    return probe_run(dev, ctx, r, { { p, x } }, { { r, out } });
}

// out (f32, packed) = ggml_step(x), x f32 packed of extents ne
int probe_step(const char * dev, const int64_t * ne, const void * x, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * tx = packed(ctx, GGML_TYPE_F32, ne);
    ggml_tensor * r = ggml_step(ctx, tx);
    return probe_run(dev, ctx, r, { { tx, x } }, { { r, out } });
}

} // extern "C"
