// oracle/sam_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_WIN_PART, GGML_OP_WIN_UNPART, GGML_OP_GET_REL_POS, GGML_OP_ADD_REL_POS, GGML_OP_CONV_TRANSPOSE_2D, GGML_OP_SIN and
// GGML_OP_COS graphs on a named device, through the UNMODIFIED reference's public API (ggml_win_part / ggml_win_unpart / ggml_get_rel_pos /
// ggml_add_rel_pos[_inplace] / ggml_conv_transpose_2d_p0 / ggml_sin / ggml_cos, ggml_backend_*), built into oracle/_ref/libggml_sam_probe.so
// and driven from Python with ctypes (oracle/sam.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with
// probe_load_backend of libggml_probe.so) it is this repository's kernel.  Nothing here is on the product path.

#include "probe_harness.h"

extern "C" {

// Every probe returns probe_run's code (probe_harness.h); its sources are probe_view_source's.

// out (f32, packed [C, w, w, npx npy]) = ggml_win_part(source, w)
int probe_win_part(const char * dev, const int64_t * spec, int w, const void * data, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = probe_view_source(ctx, spec, &parent);
    ggml_tensor * r = ggml_win_part(ctx, x, w);
    return probe_run(dev, ctx, r, { { parent, data } }, { { r, out } });
}

// out (f32, packed [C, w0, h0]) = ggml_win_unpart(source, w0, h0, w)
int probe_win_unpart(const char * dev, const int64_t * spec, int w0, int h0, int w, const void * data, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = probe_view_source(ctx, spec, &parent);
    ggml_tensor * r = ggml_win_unpart(ctx, x, w0, h0, w);
    return probe_run(dev, ctx, r, { { parent, data } }, { { r, out } });
}

// out (f16, packed [C, w, w]) = ggml_get_rel_pos(source, w, w)
int probe_get_rel_pos(const char * dev, const int64_t * spec, int w, const void * data, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = probe_view_source(ctx, spec, &parent);
    ggml_tensor * r = ggml_get_rel_pos(ctx, x, w, w);
    return probe_run(dev, ctx, r, { { parent, data } }, { { r, out } });
}

// out (f32, packed like a) = ggml_add_rel_pos[_inplace](a, pw, ph)
int probe_add_rel_pos(const char * dev, const int64_t * spec_a, const int64_t * spec_pw, const int64_t * spec_ph, int inplace,
                      const void * data_a, const void * data_pw, const void * data_ph, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * pa, * pw, * ph;
    ggml_tensor * a = probe_view_source(ctx, spec_a, &pa), * w = probe_view_source(ctx, spec_pw, &pw),
                * h = probe_view_source(ctx, spec_ph, &ph);
    ggml_tensor * r = inplace ? ggml_add_rel_pos_inplace(ctx, a, w, h) : ggml_add_rel_pos(ctx, a, w, h);
    return probe_run(dev, ctx, r, { { pa, data_a }, { pw, data_pw }, { ph, data_ph } }, { { r, out } });
}

// out (f32, packed [(W-1) s + Kw, (H-1) s + Kh, Cout, N]) = ggml_conv_transpose_2d_p0(kernel, input, stride)
int probe_conv_transpose_2d(const char * dev, const int64_t * spec_k, const int64_t * spec_x, int stride, const void * data_k, const void * data_x,
                            void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * pk, * px;
    ggml_tensor * k = probe_view_source(ctx, spec_k, &pk), * x = probe_view_source(ctx, spec_x, &px);
    ggml_tensor * r = ggml_conv_transpose_2d_p0(ctx, k, x, stride);
    return probe_run(dev, ctx, r, { { pk, data_k }, { px, data_x } }, { { r, out } });
}

// out (f32, packed like the source) = ggml_sin(source) (op 0) or ggml_cos(source) (op 1)
int probe_sin_cos(const char * dev, const int64_t * spec, int op, const void * data, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = probe_view_source(ctx, spec, &parent);
    ggml_tensor * r = op == 0 ? ggml_sin(ctx, x) : ggml_cos(ctx, x);
    return probe_run(dev, ctx, r, { { parent, data } }, { { r, out } });
}

} // extern "C"
