// oracle/core_probe.cpp — TEST INFRASTRUCTURE ONLY.
//
// The small ops either side of every mat-mul (GET_ROWS, ADD / SUB / MUL / DIV, NORM / RMS_NORM, SCALE, DIAG_MASK_INF, the UNARY functions,
// SQR / SQRT / SIN / COS, the float CPY / CONT / DUP) and the two chains the plug-in fuses (NORM -> MUL -> ADD, SCALE -> DIAG_MASK_INF ->
// SOFT_MAX) as graphs on a named device, through the UNMODIFIED reference's public API, built into oracle/_ref/libggml_core_probe.so and
// driven from Python with ctypes (oracle/core.py).  On "CPU" it is ggml-cpu's op; on "B2000" (the plug-in, loaded beforehand with
// probe_load_backend of libggml_probe.so) it is this repository's kernel.  Nothing here is on the product path.

#include "probe_harness.h"

extern "C" {

// Every probe returns probe_run's code (probe_harness.h); its sources are probe_view_source's.

// out (f32, packed [ne0, n, ne11, ne12]) = ggml_get_rows(src, ids): ids (i32) [n, ne11, ne12] selects rows of src [ne0, rows, ne11, ne12]
int probe_get_rows(const char * dev, const int64_t * spec_src, const int64_t * spec_ids, const void * data_src, const void * data_ids, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * ps, * pi;
    ggml_tensor * s = probe_view_source(ctx, spec_src, &ps), * ids = probe_view_source(ctx, spec_ids, &pi);
    ggml_tensor * r = ggml_get_rows(ctx, s, ids);
    return probe_run(dev, ctx, r, { { ps, data_src }, { pi, data_ids } }, { { r, out } });
}

// op 0 ADD, 1 MUL, 2 SUB, 3 DIV of src0 and src1 (a whole repeat of it broadcast over src0).  Not in place: out is the packed result; in place:
// the result is written into src0's view, and out receives all of src0's parent
int probe_binary(const char * dev, int op, const int64_t * spec0, const int64_t * spec1, int inplace, const void * data0, const void * data1,
                 void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * p0, * p1;
    ggml_tensor * a = probe_view_source(ctx, spec0, &p0), * b = probe_view_source(ctx, spec1, &p1);
    ggml_tensor * (* const fn[2][4])(ggml_context *, ggml_tensor *, ggml_tensor *) = {
        { ggml_add, ggml_mul, ggml_sub, ggml_div }, { ggml_add_inplace, ggml_mul_inplace, ggml_sub_inplace, ggml_div_inplace } };
    ggml_tensor * r = fn[inplace ? 1 : 0][op](ctx, a, b);
    return probe_run(dev, ctx, r, { { p0, data0 }, { p1, data1 } }, { { inplace ? p0 : r, out } });
}

// out (f32, packed) = ggml_norm (rms 0) or ggml_rms_norm (rms 1) of src with eps
int probe_norm(const char * dev, int rms, float eps, const int64_t * spec, const void * data, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * p;
    ggml_tensor * s = probe_view_source(ctx, spec, &p);
    ggml_tensor * r = rms ? ggml_rms_norm(ctx, s, eps) : ggml_norm(ctx, s, eps);
    return probe_run(dev, ctx, r, { { p, data } }, { { r, out } });
}

// out (f32, packed) = a unary function of src, by the kernel library's code (GGML_B200_UNARY_*): 0 GELU, 1 SILU, 2 RELU, 3 TANH, 4 NEG,
// 5 ABS, 6 GELU_QUICK, 7 SIGMOID, 8 EXP, 9 SQR, 10 SQRT, 11 SIN, 12 COS, 13 STEP (9-12 are ops of their own, the rest GGML_OP_UNARY)
int probe_unary(const char * dev, int code, const int64_t * spec, const void * data, void * out) {
    ggml_tensor * (* const fn[14])(ggml_context *, ggml_tensor *) = { ggml_gelu, ggml_silu, ggml_relu, ggml_tanh, ggml_neg, ggml_abs,
        ggml_gelu_quick, ggml_sigmoid, ggml_exp, ggml_sqr, ggml_sqrt, ggml_sin, ggml_cos, ggml_step };
    if (code < 0 || code > 13) return -5;
    ggml_context * ctx = probe_ctx();
    ggml_tensor * p;
    ggml_tensor * s = probe_view_source(ctx, spec, &p);
    ggml_tensor * r = fn[code](ctx, s);
    return probe_run(dev, ctx, r, { { p, data } }, { { r, out } });
}

// the two-node graph ggml_diag_mask_inf(ggml_scale(a, scale), n_past) of a packed f32 a: out_scaled and out_masked (both packed) receive
// the two nodes.  No SOFT_MAX follows, so the plug-in runs each node on its own
int probe_scale_mask(const char * dev, const int64_t * ne, float scale, int n_past, const void * data, void * out_scaled, void * out_masked) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * a = ggml_new_tensor(ctx, GGML_TYPE_F32, 4, ne);
    ggml_tensor * s = ggml_scale(ctx, a, scale);
    ggml_tensor * r = ggml_diag_mask_inf(ctx, s, n_past);
    return probe_run(dev, ctx, r, { { a, data } }, { { s, out_scaled }, { r, out_masked } });
}

// op 0: ggml_cpy(src, dst view) into a float parent of any type filled from dst_in first, out receiving all of that parent's bytes;
// op 1 / 2: ggml_cont / ggml_dup(src), out receiving the packed result (src's type; spec_dst is not read)
int probe_cpy(const char * dev, int op, const int64_t * spec_src, const int64_t * spec_dst, const void * data_src, const void * dst_in, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * ps, * pd = nullptr;
    ggml_tensor * s = probe_view_source(ctx, spec_src, &ps);
    ggml_tensor * r = op == 0 ? ggml_cpy(ctx, s, probe_view_source(ctx, spec_dst, &pd)) : op == 1 ? ggml_cont(ctx, s) : ggml_dup(ctx, s);
    return probe_run(dev, ctx, r, { { ps, data_src }, { pd, dst_in } }, { { op == 0 ? pd : r, out } });
}

// the three-node graph ggml_add(ggml_mul(norm(a), gain), bias), norm = ggml_norm (rms 0) or ggml_rms_norm (rms 1) with eps, of a packed
// f32 a [ne] and f32 row vectors gain and bias [ne[0]] (the plug-in fuses it); out_norm, out_mul and out_add receive the three nodes
int probe_norm_affine(const char * dev, int rms, float eps, const int64_t * ne, const void * data, const void * gain, const void * bias,
                      void * out_norm, void * out_mul, void * out_add) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * a = ggml_new_tensor(ctx, GGML_TYPE_F32, 4, ne);
    ggml_tensor * g = ggml_new_tensor_1d(ctx, GGML_TYPE_F32, ne[0]), * b = ggml_new_tensor_1d(ctx, GGML_TYPE_F32, ne[0]);
    ggml_tensor * n = rms ? ggml_rms_norm(ctx, a, eps) : ggml_norm(ctx, a, eps);
    ggml_tensor * m = ggml_mul(ctx, n, g);
    ggml_tensor * r = ggml_add(ctx, m, b);
    return probe_run(dev, ctx, r, { { a, data }, { g, gain }, { b, bias } }, { { n, out_norm }, { m, out_mul }, { r, out_add } });
}

// out (f32, packed) = ggml_soft_max(ggml_diag_mask_inf(ggml_scale(a, scale), n_past)) of a packed f32 a (the plug-in fuses the three nodes
// and does not write the two intermediates, so only the result is read)
int probe_scale_mask_softmax(const char * dev, const int64_t * ne, float scale, int n_past, const void * data, void * out) {
    ggml_context * ctx = probe_ctx();
    ggml_tensor * a = ggml_new_tensor(ctx, GGML_TYPE_F32, 4, ne);
    ggml_tensor * r = ggml_soft_max(ctx, ggml_diag_mask_inf(ctx, ggml_scale(ctx, a, scale), n_past));
    return probe_run(dev, ctx, r, { { a, data } }, { { r, out } });
}

} // extern "C"
