// oracle/pool_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_POOL_2D, GGML_OP_UPSCALE, GGML_OP_LEAKY_RELU and GGML_OP_REPEAT graphs on a named device, through the UNMODIFIED
// reference's public API (ggml_pool_2d / ggml_upscale_ext / ggml_leaky_relu / ggml_repeat, ggml_backend_*), built into
// oracle/_ref/libggml_pool_probe.so and driven from Python with ctypes (oracle/pool.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the
// plug-in, loaded beforehand with probe_load_backend of libggml_probe.so) it is this repository's kernel.  Nothing here is on the product path.

#include "probe_harness.h"

extern "C" {

// Every probe returns probe_run's code (probe_harness.h); its source is probe_view_source's.

// out (f32, packed [OW, OH, C, N]) = ggml_pool_2d(source, op, k0, k1, s0, s1, p0, p1) with ggml_pool_2d's float paddings
int probe_pool_2d(const char * dev, const int64_t * spec, int op, int k0, int k1, int s0, int s1, float p0, float p1, const void * data, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = probe_view_source(ctx, spec, &parent);
    ggml_tensor * r = ggml_pool_2d(ctx, x, (ggml_op_pool) op, k0, k1, s0, s1, p0, p1);
    return probe_run(dev, ctx, r, { { parent, data } }, { { r, out } });
}

// out (f32, packed ne) = ggml_upscale_ext(source, ne)
int probe_upscale(const char * dev, const int64_t * spec, const int64_t * ne, const void * data, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = probe_view_source(ctx, spec, &parent);
    ggml_tensor * r = ggml_upscale_ext(ctx, x, (int) ne[0], (int) ne[1], (int) ne[2], (int) ne[3]);
    return probe_run(dev, ctx, r, { { parent, data } }, { { r, out } });
}

// out = ggml_leaky_relu(source, slope, inplace); in place the result is the source view itself, so out receives ggml_nbytes of it (a
// packed source gives the packed result)
int probe_leaky_relu(const char * dev, const int64_t * spec, float slope, int inplace, const void * data, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = probe_view_source(ctx, spec, &parent);
    ggml_tensor * r = ggml_leaky_relu(ctx, x, slope, inplace != 0);
    return probe_run(dev, ctx, r, { { parent, data } }, { { r, out } });
}

// out (the source's type, packed ne) = ggml_repeat(source, a tensor of shape ne)
int probe_repeat(const char * dev, const int64_t * spec, const int64_t * ne, const void * data, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = probe_view_source(ctx, spec, &parent);
    ggml_tensor * r = ggml_repeat(ctx, x, ggml_new_tensor(ctx, x->type, 4, ne));
    return probe_run(dev, ctx, r, { { parent, data } }, { { r, out } });
}

} // extern "C"
