// oracle/attn_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_FLASH_ATTN_EXT, GGML_OP_SOFT_MAX and GGML_OP_CPY graphs on a named device, through the UNMODIFIED reference's public API
// (ggml_flash_attn_ext / ggml_soft_max_ext / ggml_cpy, ggml_backend_*), built into oracle/_ref/libggml_attn_probe.so and driven from Python
// with ctypes (oracle/attn.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with probe_load_backend of
// libggml_probe.so) it is this repository's kernel.  Nothing here is on the product path.

#include "probe_harness.h"

extern "C" {

// Every probe returns probe_run's code (probe_harness.h); its sources are probe_view_source's.

// out (f32, packed [D, n_head, n_q, ne3]) = ggml_flash_attn_ext(q, k, v, mask, scale, max_bias, softcap).  K and V are views of their cache
// parents (any type); q is read through ggml_permute(q, 0, 2, 1, 3) when permute_q (its spec then describes the unpermuted [D, n_head, n_q,
// ne3]); mask_rows > 0: an f16 mask [ne0 of K's view, mask_rows] (a multiple of GGML_KQ_MASK_PAD), none otherwise.
int probe_flash_attn_ext(const char * dev, const int64_t * spec_q, int permute_q, const int64_t * spec_k, const int64_t * spec_v, int64_t mask_rows,
                         float scale, float max_bias, float softcap, const void * data_q, const void * data_k, const void * data_v,
                         const void * data_mask, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * pq, * pk, * pv;
    ggml_tensor * q = probe_view_source(ctx, spec_q, &pq), * k = probe_view_source(ctx, spec_k, &pk), * v = probe_view_source(ctx, spec_v, &pv);
    if (permute_q) q = ggml_permute(ctx, q, 0, 2, 1, 3);
    ggml_tensor * mask = mask_rows > 0 ? ggml_new_tensor_2d(ctx, GGML_TYPE_F16, k->ne[1], mask_rows) : nullptr;
    ggml_tensor * r = ggml_flash_attn_ext(ctx, q, k, v, mask, scale, max_bias, softcap);
    return probe_run(dev, ctx, r, { { pq, data_q }, { pk, data_k }, { pv, data_v }, { mask, data_mask } }, { { r, out } });
}

// out (f32, packed ne[4]) = ggml_soft_max_ext(a, mask, scale, max_bias) of a packed f32 a; mask_type 0 (f32) or 1 (f16) [ne0, mask_rows],
// mask_type < 0: none
int probe_soft_max(const char * dev, const int64_t * ne, int mask_type, int64_t mask_rows, float scale, float max_bias, const void * data_a,
                   const void * data_mask, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * a = ggml_new_tensor(ctx, GGML_TYPE_F32, 4, ne);
    ggml_tensor * mask = mask_type >= 0 ? ggml_new_tensor_2d(ctx, (ggml_type) mask_type, ne[0], mask_rows) : nullptr;
    ggml_tensor * r = ggml_soft_max_ext(ctx, a, mask, scale, max_bias);
    return probe_run(dev, ctx, r, { { a, data_a }, { mask, data_mask } }, { { r, out } });
}

// ggml_cpy(source, view of a cache): the f32 source (spec_src) into the view spec_dst describes of a cache parent of any type; the cache is
// filled from cache_in first, and all of its bytes are read back into cache_out
int probe_cpy(const char * dev, const int64_t * spec_src, const int64_t * spec_dst, const void * data_src, const void * cache_in, void * cache_out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * ps, * pc;
    ggml_tensor * s = probe_view_source(ctx, spec_src, &ps), * d = probe_view_source(ctx, spec_dst, &pc);
    ggml_tensor * r = ggml_cpy(ctx, s, d);
    return probe_run(dev, ctx, r, { { ps, data_src }, { pc, cache_in } }, { { pc, cache_out } });
}

} // extern "C"
