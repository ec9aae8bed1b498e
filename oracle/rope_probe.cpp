// oracle/rope_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_ROPE graphs on a named device, through the UNMODIFIED reference's public API (ggml_rope_ext /
// ggml_rope_ext_inplace / ggml_rope_multi, ggml_backend_*), built into oracle/_ref/libggml_rope_probe.so and driven from Python with
// ctypes.  On "CPU" it is ggml-cpu's ROPE; on "B2000" (the plug-in, loaded beforehand with probe_load_backend of libggml_probe.so:
// both libraries share the reference's backend registry) it is this repository's kernel.  Nothing here is on the product path.

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

#include <cstring>

extern "C" {

// out = ROPE(x) on device `dev`.  ne: the shape roped.  view != 0: x holds a parent tensor of shape ne * {2, 4, 3, 1} and the rope reads
// its ne-shaped corner through a strided view (what tests/test-backend-ops.cpp's test_rope does with v = 1).  inplace != 0: the in-place
// form (ggml_rope_ext_inplace: the result aliases x; NORM / NEOX only).  MROPE / VISION (mode & 8) go through ggml_rope_multi.
// pos: ne[2] positions (4 * ne[2] for MROPE / VISION); ff: NULL or n_ff freq factors.  out: the result, contiguous.
// Returns 0, -1 (no such device), -2 (the device declines the node), -3 (allocation failed).
int probe_rope(const char * dev, int type, const int64_t * ne, int view, int inplace, const void * x, const int32_t * pos, const float * ff, int64_t n_ff,
               int n_dims, int mode, const int32_t * sections, int n_ctx_orig, float freq_base, float freq_scale, float ext_factor, float attn_factor,
               float beta_fast, float beta_slow, void * out) {
    ggml_backend_dev_t d = ggml_backend_dev_by_name(dev);
    if (!d) return -1;
    ggml_backend_t be = ggml_backend_dev_init(d, nullptr);
    if (!be) return -1;
    if (ggml_backend_is_cpu(be)) ggml_backend_cpu_set_n_threads(be, 4);
    ggml_init_params ip = { ggml_tensor_overhead() * 16 + ggml_graph_overhead(), nullptr, true };
    ggml_context * ctx = ggml_init(ip);
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
    ggml_cgraph * gf = ggml_new_graph(ctx);
    ggml_build_forward_expand(gf, r);
    int rc = 0;
    ggml_backend_buffer_t buf = nullptr;
    if (!ggml_backend_supports_op(be, r)) rc = -2;
    else if (!(buf = ggml_backend_alloc_ctx_tensors(ctx, be))) rc = -3;
    else {
        ggml_backend_tensor_set(parent, x, 0, ggml_nbytes(parent));
        ggml_backend_tensor_set(p, pos, 0, ggml_nbytes(p));
        if (f) ggml_backend_tensor_set(f, ff, 0, ggml_nbytes(f));
        ggml_backend_graph_compute(be, gf);
        ggml_backend_tensor_get(r, out, 0, ggml_nbytes(r));
    }
    if (buf) ggml_backend_buffer_free(buf);
    ggml_free(ctx);
    ggml_backend_free(be);
    return rc;
}

} // extern "C"
