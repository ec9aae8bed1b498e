// oracle/rope_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_ROPE graphs on a named device, through the UNMODIFIED reference's public API (ggml_rope_ext /
// ggml_rope_ext_inplace / ggml_rope_multi, ggml_backend_*), built into oracle/_ref/libggml_rope_probe.so and driven from Python with
// ctypes.  On "CPU" it is ggml-cpu's ROPE; on "B2000" (the plug-in, loaded beforehand with probe_load_backend of libggml_probe.so:
// both libraries share the reference's backend registry) it is this repository's kernel.  Nothing here is on the product path.

#include "probe_harness.h"

extern "C" {

// out = ROPE(x) on device `dev`.  ne: the shape roped.  view != 0: x holds a parent tensor of shape ne * {2, 4, 3, 1} and the rope reads
// its ne-shaped corner through a strided view (what tests/test-backend-ops.cpp's test_rope does with v = 1).  inplace != 0: the in-place
// form (ggml_rope_ext_inplace: the result aliases x; NORM / NEOX only).  MROPE / VISION (mode & 8) go through ggml_rope_multi.
// pos: ne[2] positions (4 * ne[2] for MROPE / VISION); ff: NULL or n_ff freq factors.  out: the result, contiguous.
// Returns probe_run's code (probe_harness.h).
int probe_rope(const char * dev, int type, const int64_t * ne, int view, int inplace, const void * x, const int32_t * pos, const float * ff, int64_t n_ff,
               int n_dims, int mode, const int32_t * sections, int n_ctx_orig, float freq_base, float freq_scale, float ext_factor, float attn_factor,
               float beta_fast, float beta_slow, void * out) {
    ggml_context * ctx = probe_ctx();
    const bool multi = (mode & GGML_ROPE_TYPE_MROPE) != 0;
    ggml_tensor * parent, * a;
    if (view) {
        parent = ggml_new_tensor_4d(ctx, (ggml_type) type, ne[0] * 2, ne[1] * 4, ne[2] * 3, ne[3]);
        a = ggml_view_4d(ctx, parent, ne[0], ne[1], ne[2], ne[3], parent->nb[1], parent->nb[2], parent->nb[3], 0);
    } else {
        parent = a = ggml_new_tensor_4d(ctx, (ggml_type) type, ne[0], ne[1], ne[2], ne[3]);
    }
    ggml_tensor * p = ggml_new_tensor_1d(ctx, GGML_TYPE_I32, ne[2] * (multi ? 4 : 1));
    ggml_tensor * f = ff ? ggml_new_tensor_1d(ctx, GGML_TYPE_F32, n_ff) : nullptr;
    ggml_tensor * r;
    if (multi) {
        int s[4] = { sections[0], sections[1], sections[2], sections[3] };
        r = ggml_rope_multi(ctx, a, p, f, n_dims, s, mode, n_ctx_orig, freq_base, freq_scale, ext_factor, attn_factor, beta_fast, beta_slow);
    } else if (inplace) {
        r = ggml_rope_ext_inplace(ctx, a, p, f, n_dims, mode, n_ctx_orig, freq_base, freq_scale, ext_factor, attn_factor, beta_fast, beta_slow);
    } else {
        r = ggml_rope_ext(ctx, a, p, f, n_dims, mode, n_ctx_orig, freq_base, freq_scale, ext_factor, attn_factor, beta_fast, beta_slow);
    }
    return probe_run(dev, ctx, r, { { parent, x }, { p, pos }, { f, ff } }, { { r, out } });
}

} // extern "C"
