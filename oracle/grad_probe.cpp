// oracle/grad_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// MUL_MAT's backward graph on a named device, as the reference's test-backend-ops builds and checks it, through the UNMODIFIED
// reference's public API (ggml_mul_mat / ggml_sum / ggml_build_backward_expand / ggml_graph_reset, ggml_backend_*), built into
// oracle/_ref/libggml_grad_probe.so by oracle/grad.mk and driven from Python with ctypes (oracle/grad.py).  On "CPU" it is ggml-cpu; on
// "B2000" (the plug-in, loaded beforehand with probe_load_backend of libggml_probe.so) it is this repository's kernels.  Nothing here is
// on the product path.

#include "probe_harness.h"

#include <algorithm>

extern "C" {

// MUL_MAT's gradient as the reference's test-backend-ops checks it (test_mul_mat::build_graph and test_case::eval_grad): parents a
// [k, m, bs0, bs1] and b [k, n, bs0 nr0, bs1 nr1], each created with its extents permuted by per and permuted back; a is a parameter only
// when bs1 == nr1 == 1, b always; loss = ggml_sum(ggml_mul_mat(a, b)); the backward graph of ggml_build_backward_expand.  cfg (int64):
// m, n, k, bs0, bs1, nr0, nr1, per[4].  a and b are the parents' f32 data as created (per-permuted extents, packed).
// Writes the loss of the forward graph to *loss and each parameter's gradient, read element by element in its parent's layout, to ga_a
// (a not a parameter: left untouched) and ga_b.  Then, for each of the n_ia linear indices ia of a (n_ib, ib of b), the numerical gradient
// of test-backend-ops' two-point procedure: x0 +- eps set as f32, the forward graph recomputed, (fu - fd) / (2 eps) in float, x0 restored.
// Every tensor that is not an input or a view starts NaN, so a kernel that reads its destination before writing it shows.
// Returns probe_run's codes; -5: gn asked of a, which is not a parameter.
int probe_mul_mat_grad(const char * dev, const int64_t * cfg, const void * a, const void * b, float eps, float * loss, void * ga_a, void * ga_b,
                       int64_t n_ia, const int64_t * ia, float * gn_a, int64_t n_ib, const int64_t * ib, float * gn_b) {
    const int64_t m = cfg[0], n = cfg[1], k = cfg[2], bs0 = cfg[3], bs1 = cfg[4], nr0 = cfg[5], nr1 = cfg[6];
    const int64_t * per = cfg + 7;
    const bool a_param = bs1 == 1 && nr1 == 1;
    if (n_ia > 0 && !a_param) return -5;
    ggml_backend_dev_t d = ggml_backend_dev_by_name(dev);
    ggml_backend_t be = d ? ggml_backend_dev_init(d, nullptr) : nullptr;
    if (!be) return -1;
    if (ggml_backend_is_cpu(be)) ggml_backend_cpu_set_n_threads(be, 1);     // thousands of small graphs: no thread start per compute
    ggml_init_params ip = { ggml_tensor_overhead() * 128 + 2 * ggml_graph_overhead_custom(GGML_DEFAULT_GRAPH_SIZE, true), nullptr, true };
    ggml_context * ctx = ggml_init(ip);
    ggml_cgraph * gf = ggml_new_graph_custom(ctx, GGML_DEFAULT_GRAPH_SIZE, true), * gb = ggml_new_graph_custom(ctx, GGML_DEFAULT_GRAPH_SIZE, true);
    const int64_t ne_a[4] = { k, m, bs0, bs1 }, ne_b[4] = { k, n, bs0 * nr0, bs1 * nr1 };
    ggml_tensor * ta = ggml_new_tensor_4d(ctx, GGML_TYPE_F32, ne_a[per[0]], ne_a[per[1]], ne_a[per[2]], ne_a[per[3]]);
    ggml_tensor * tb = ggml_new_tensor_4d(ctx, GGML_TYPE_F32, ne_b[per[0]], ne_b[per[1]], ne_b[per[2]], ne_b[per[3]]);
    if (a_param) ggml_set_param(ctx, ta);
    ggml_set_param(ctx, tb);
    const bool permuted = per[0] != 0 || per[1] != 1 || per[2] != 2 || per[3] != 3;
    ggml_tensor * va = permuted ? ggml_permute(ctx, ta, per[0], per[1], per[2], per[3]) : ta;
    ggml_tensor * vb = permuted ? ggml_permute(ctx, tb, per[0], per[1], per[2], per[3]) : tb;
    ggml_tensor * out = ggml_sum(ctx, ggml_mul_mat(ctx, va, vb));
    ggml_set_loss(out);
    ggml_build_forward_expand(gf, out);
    ggml_graph_cpy(gf, gb);
    ggml_build_backward_expand(ctx, ctx, gb, false);

    int rc = 0;
    for (ggml_tensor * t = ggml_get_first_tensor(ctx); t; t = ggml_get_next_tensor(ctx, t))
        if (!ggml_backend_supports_op(be, t)) rc = -2;
    ggml_backend_buffer_t buf = nullptr;
    if (rc == 0 && !(buf = ggml_backend_alloc_ctx_tensors(ctx, be))) rc = -3;
    if (rc == 0) {
        for (ggml_tensor * t = ggml_get_first_tensor(ctx); t; t = ggml_get_next_tensor(ctx, t)) {
            if (t == ta || t == tb || t->view_src) continue;
            std::vector<uint32_t> nan(ggml_nbytes(t) / 4, 0x7fc00000u);
            ggml_backend_tensor_set(t, nan.data(), 0, ggml_nbytes(t));
        }
        ggml_backend_tensor_set(ta, a, 0, ggml_nbytes(ta));
        ggml_backend_tensor_set(tb, b, 0, ggml_nbytes(tb));
        ggml_graph_reset(gb);
        if (ggml_backend_graph_compute(be, gf) != GGML_STATUS_SUCCESS || ggml_backend_graph_compute(be, gb) != GGML_STATUS_SUCCESS) rc = -4;
    }
    if (rc == 0) {
        ggml_backend_tensor_get(out, loss, 0, sizeof(float));
        const std::pair<ggml_tensor *, void *> params[2] = { { a_param ? ta : nullptr, ga_a }, { tb, ga_b } };
        for (const auto & p : params) {
            if (!p.first) continue;
            float * dst = (float *) p.second;
            const ggml_tensor * g = ggml_graph_get_grad(gb, p.first);
            if (!g) { std::fill(dst, dst + ggml_nelements(p.first), 0.0f); continue; }
            std::vector<uint8_t> raw(ggml_nbytes(g));
            ggml_backend_tensor_get(g, raw.data(), 0, raw.size());
            for (int64_t i3 = 0; i3 < g->ne[3]; ++i3) for (int64_t i2 = 0; i2 < g->ne[2]; ++i2) for (int64_t i1 = 0; i1 < g->ne[1]; ++i1)
                for (int64_t i0 = 0; i0 < g->ne[0]; ++i0)
                    *dst++ = *(const float *) &raw[i3 * g->nb[3] + i2 * g->nb[2] + i1 * g->nb[1] + i0 * g->nb[0]];
        }
        const struct { ggml_tensor * t; const void * x0; int64_t n; const int64_t * idx; float * gn; } fd[2] = {
            { ta, a, n_ia, ia, gn_a }, { tb, b, n_ib, ib, gn_b } };
        for (const auto & p : fd) {
            for (int64_t j = 0; j < p.n && rc == 0; ++j) {
                const float x0 = ((const float *) p.x0)[p.idx[j]], xu = x0 + 1.0f * eps, xd = x0 - 1.0f * eps;
                float fu, fdn;
                ggml_backend_tensor_set(p.t, &xu, p.idx[j] * sizeof(float), sizeof(float));
                if (ggml_backend_graph_compute(be, gf) != GGML_STATUS_SUCCESS) rc = -4;
                ggml_backend_tensor_get(out, &fu, 0, sizeof(float));
                ggml_backend_tensor_set(p.t, &xd, p.idx[j] * sizeof(float), sizeof(float));
                if (ggml_backend_graph_compute(be, gf) != GGML_STATUS_SUCCESS) rc = -4;
                ggml_backend_tensor_get(out, &fdn, 0, sizeof(float));
                p.gn[j] = (fu - fdn) / (2.0f * eps);
                ggml_backend_tensor_set(p.t, p.x0, 0, ggml_nbytes(p.t));
            }
        }
    }
    if (buf) ggml_backend_buffer_free(buf);
    ggml_free(ctx);
    ggml_backend_free(be);
    return rc;
}

} // extern "C"
