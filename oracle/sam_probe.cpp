// oracle/sam_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// One-node GGML_OP_WIN_PART, GGML_OP_WIN_UNPART, GGML_OP_GET_REL_POS, GGML_OP_ADD_REL_POS, GGML_OP_CONV_TRANSPOSE_2D, GGML_OP_SIN and
// GGML_OP_COS graphs on a named device, through the UNMODIFIED reference's public API (ggml_win_part / ggml_win_unpart / ggml_get_rel_pos /
// ggml_add_rel_pos[_inplace] / ggml_conv_transpose_2d_p0 / ggml_sin / ggml_cos, ggml_backend_*), built into oracle/_ref/libggml_sam_probe.so
// and driven from Python with ctypes (oracle/sam.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with
// probe_load_backend of libggml_probe.so) it is this repository's kernel.  Nothing here is on the product path.

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

#include <vector>

namespace {

// A source of a probe, read through a view of its own parent.  spec (int64): type, the parent's ne[4], the view's ne[4], its nb1, nb2, nb3
// (bytes), its byte offset, and 1 to read the view transposed (dims 0 and 1 swapped, ggml_transpose) -- oracle/pool.py's Source.spec()
ggml_tensor * source(ggml_context * ctx, const int64_t * spec, ggml_tensor ** parent) {
    ggml_tensor * p = ggml_new_tensor(ctx, (ggml_type) spec[0], 4, spec + 1);
    *parent = p;
    ggml_tensor * v = ggml_view_4d(ctx, p, spec[5], spec[6], spec[7], spec[8], (size_t) spec[9], (size_t) spec[10], (size_t) spec[11], (size_t) spec[12]);
    return spec[13] ? ggml_transpose(ctx, v) : v;
}

// build the graph of `r` and run it on `dev` (every node must be supported); data[i] fills parents[i], out receives r (its ggml_nbytes)
int run(const char * dev, ggml_context * ctx, const std::vector<ggml_tensor *> & parents, const std::vector<const void *> & data, ggml_tensor * r, void * out) {
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
        else ggml_backend_tensor_get(r, out, 0, ggml_nbytes(r));
    }
    if (buf) ggml_backend_buffer_free(buf);
    ggml_free(ctx);
    ggml_backend_free(be);
    return rc;
}

ggml_context * new_ctx() {
    ggml_init_params ip = { ggml_tensor_overhead() * 24 + ggml_graph_overhead(), nullptr, true };
    return ggml_init(ip);
}

} // namespace

extern "C" {

// Every probe returns 0, -1 (no such device), -2 (the device declines a node), -3 (allocation failed) or -4 (compute failed).

// out (f32, packed [C, w, w, npx npy]) = ggml_win_part(source, w)
int probe_win_part(const char * dev, const int64_t * spec, int w, const void * data, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = source(ctx, spec, &parent);
    return run(dev, ctx, { parent }, { data }, ggml_win_part(ctx, x, w), out);
}

// out (f32, packed [C, w0, h0]) = ggml_win_unpart(source, w0, h0, w)
int probe_win_unpart(const char * dev, const int64_t * spec, int w0, int h0, int w, const void * data, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = source(ctx, spec, &parent);
    return run(dev, ctx, { parent }, { data }, ggml_win_unpart(ctx, x, w0, h0, w), out);
}

// out (f16, packed [C, w, w]) = ggml_get_rel_pos(source, w, w)
int probe_get_rel_pos(const char * dev, const int64_t * spec, int w, const void * data, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = source(ctx, spec, &parent);
    return run(dev, ctx, { parent }, { data }, ggml_get_rel_pos(ctx, x, w, w), out);
}

// out (f32, packed like a) = ggml_add_rel_pos[_inplace](a, pw, ph)
int probe_add_rel_pos(const char * dev, const int64_t * spec_a, const int64_t * spec_pw, const int64_t * spec_ph, int inplace,
                      const void * data_a, const void * data_pw, const void * data_ph, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * pa, * pw, * ph;
    ggml_tensor * a = source(ctx, spec_a, &pa), * w = source(ctx, spec_pw, &pw), * h = source(ctx, spec_ph, &ph);
    ggml_tensor * r = inplace ? ggml_add_rel_pos_inplace(ctx, a, w, h) : ggml_add_rel_pos(ctx, a, w, h);
    return run(dev, ctx, { pa, pw, ph }, { data_a, data_pw, data_ph }, r, out);
}

// out (f32, packed [(W-1) s + Kw, (H-1) s + Kh, Cout, N]) = ggml_conv_transpose_2d_p0(kernel, input, stride)
int probe_conv_transpose_2d(const char * dev, const int64_t * spec_k, const int64_t * spec_x, int stride, const void * data_k, const void * data_x,
                            void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * pk, * px;
    ggml_tensor * k = source(ctx, spec_k, &pk), * x = source(ctx, spec_x, &px);
    return run(dev, ctx, { pk, px }, { data_k, data_x }, ggml_conv_transpose_2d_p0(ctx, k, x, stride), out);
}

// out (f32, packed like the source) = ggml_sin(source) (op 0) or ggml_cos(source) (op 1)
int probe_sin_cos(const char * dev, const int64_t * spec, int op, const void * data, void * out) {
    ggml_context * ctx = new_ctx();
    ggml_tensor * parent;
    ggml_tensor * x = source(ctx, spec, &parent);
    return run(dev, ctx, { parent }, { data }, op == 0 ? ggml_sin(ctx, x) : ggml_cos(ctx, x), out);
}

} // extern "C"
