// b200_train.cuh — the per-element logic of the ops ggml_opt's backward and optimizer graphs add to a model's forward graph, as ggml-cpu
// computes them (src/ggml-cpu/ggml-cpu.c): OUT_PROD :7788-7905 (+ ggml_vec_mad_f32_unroll :1617), CROSS_ENTROPY_LOSS :12449-12525
// (+ ggml_vec_log_soft_max_f32 :2094), CROSS_ENTROPY_LOSS_BACK :12545-12605 (+ ggml_vec_soft_max_f32 :2041), OPT_STEP_ADAMW :12626-12685,
// ARGMAX :5773-5795 (+ ggml_vec_argmax_f32 :2171), COUNT_EQUAL :5821-5878, SUM :5537-5565, REPEAT_BACK :6019-6075, STEP :1737.
// __host__ __device__, so that tests/hostemu compiles the same code for the CPU.
//
// OPT_STEP_ADAMW, ARGMAX, COUNT_EQUAL, REPEAT_BACK and STEP are bit-identical to ggml-cpu: every arithmetic step is one correctly rounded
// IEEE operation (pool_add / pool_mul / pool_div / train_sqrt) in the CPU's order.  OUT_PROD accumulates each output with fused multiply-adds
// in ascending k, the chain of ggml-cpu's SIMD body; SUM and the cross-entropy pair reduce in a fixed order of their own.
#pragma once

#include "../../include/ggml-b200.h"
#include "b200_pool.cuh"

#include <cmath>
#include <cstdint>

namespace b200 {

__host__ __device__ __forceinline__ float train_sqrt(float a) {
#ifdef __CUDA_ARCH__
    return __fsqrt_rn(a);
#else
    return std::sqrt(a);
#endif
}

// --------------------------------------------------------------------------------------------- OPT_STEP_ADAMW
// The seven hyper-parameters in ggml_opt's order (ggml-opt.cpp, ggml_opt_get_default_optimizer_params / ggml_opt_eval): alpha, beta1, beta2,
// eps, wd, beta1h = 1 / (1 - beta1^t), beta2h = 1 / (1 - beta2^t).
enum { ADAMW_ALPHA = 0, ADAMW_BETA1, ADAMW_BETA2, ADAMW_EPS, ADAMW_WD, ADAMW_BETA1H, ADAMW_BETA2H, ADAMW_NPARAMS };

// One element, each line of ggml-cpu's loop spelled out in C's evaluation order (no contraction):
//   m = m*beta1 + g*(1 - beta1);  v = v*beta2 + g*g*(1 - beta2);  mh = m*beta1h;  vh = sqrtf(v*beta2h) + eps;
//   w = w*(1 - alpha*wd) - alpha*mh/vh   (alpha*mh/vh is (alpha*mh)/vh)
__host__ __device__ __forceinline__ void adamw_update(float & w, float g, float & m, float & v, const float * p) {
    const float alpha = p[ADAMW_ALPHA], beta1 = p[ADAMW_BETA1], beta2 = p[ADAMW_BETA2], eps = p[ADAMW_EPS], wd = p[ADAMW_WD];
    m = pool_add(pool_mul(m, beta1), pool_mul(g, pool_add(1.0f, -beta1)));
    v = pool_add(pool_mul(v, beta2), pool_mul(pool_mul(g, g), pool_add(1.0f, -beta2)));
    const float mh = pool_mul(m, p[ADAMW_BETA1H]);
    const float vh = pool_add(train_sqrt(pool_mul(v, p[ADAMW_BETA2H])), eps);
    w = pool_add(pool_mul(w, pool_add(1.0f, -pool_mul(alpha, wd))), -pool_div(pool_mul(alpha, mh), vh));
}

// --------------------------------------------------------------------------------------------- ARGMAX
// ggml_vec_argmax_f32: max = -inf, idx = 0; for each i: max = MAX(max, x[i]) (a > b ? a : b); if (max == x[i]) idx = i.
// A NaN makes max NaN without taking its index, and the next element then becomes max whatever it is.  The closed form a parallel
// reduction computes: drop the trailing run of NaNs; over the elements after the last NaN that remains, the LAST index of the greatest
// value (== ties, so -0 and +0 tie); a row of NaNs only gives 0.
//
// The reduction's combine: (v, i) beats (w, j) when v > w, or v == w and i > j.  Indices of -1 stand for "nothing".
__host__ __device__ __forceinline__ bool argmax_beats(float v, int32_t i, float w, int32_t j) {
    return j < 0 || (i >= 0 && (v > w || (v == w && i > j)));
}

// the sequential rule itself, the host test's and the emulation's reference
inline int32_t argmax_row_seq(const float * x, int64_t n) {
    float max = -INFINITY;
    int32_t idx = 0;
    for (int64_t i = 0; i < n; ++i) {
        max = max > x[i] ? max : x[i];
        if (max == x[i]) idx = (int32_t)i;
    }
    return idx;
}

// the closed form, in the three passes the device kernel makes over a row
inline int32_t argmax_row_closed(const float * x, int64_t n) {
    int64_t last = -1;                                        // the last element that is not NaN
    for (int64_t i = 0; i < n; ++i) if (!std::isnan(x[i])) last = i;
    if (last < 0) return 0;
    int64_t nan_before = -1;                                  // the last NaN before it
    for (int64_t i = 0; i < last; ++i) if (std::isnan(x[i])) nan_before = i;
    float bv = 0.0f;
    int32_t bi = -1;
    for (int64_t i = nan_before + 1; i <= last; ++i) if (argmax_beats(x[i], (int32_t)i, bv, bi)) { bv = x[i]; bi = (int32_t)i; }
    return bi;
}

// --------------------------------------------------------------------------------------------- OUT_PROD
// dst[i0, i1, i2, i3] = sum over k of src0[i0, k, i2 / dps2, i3 / dps3] * src1[i1, k, i2, i3], from +0 in ascending k with one fused
// multiply-add per term: the chain ggml_vec_mad_f32_unroll's SIMD body gives each element (ne0 rounded down to a multiple of 32 on the
// AVX2 build); its scalar tail multiplies and adds separately (ggml-cpu builds with -std=c11: no contraction), which this differs from.
__host__ __device__ __forceinline__ float out_prod_step(float acc, float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmaf_rn(a, b, acc);
#else
    return std::fma(a, b, acc);
#endif
}

// The device tiling (ops.cu, out_prod_kernel): a CTA of OP_THREADS threads owns OP_BM x OP_BN outputs (i0 x i1) of one (i2, i3) and walks
// K in slices of OP_BK, staging both operands' slices in shared memory; each thread keeps OP_TM x OP_TN accumulators.
enum { OP_BM = 128, OP_BN = 128, OP_BK = 8, OP_TM = 8, OP_TN = 8, OP_THREADS = 256 };

// --------------------------------------------------------------------------------------------- CROSS_ENTROPY_LOSS
// One row of nc logits x and labels l (ggml-cpu.c:12484-12500):  max = max x;  s = (double) sum expf(x_i - max);  lse = logf((float) s);
// term_i = ((x_i - max) + (-lse)) * l_i;  row = (float) (double) sum term_i.  The loss is -1/nr times the sum of the rows.
__host__ __device__ __forceinline__ float ce_term(float x, float max, float neg_lse, float l) {
    return pool_mul(pool_add(pool_add(x, -max), neg_lse), l);
}

// --------------------------------------------------------------------------------------------- CROSS_ENTROPY_LOSS_BACK
// One element (ggml-cpu.c:12580-12590): e = expf(x - max), inv = (float)(1.0 / s) with s the row's double sum of e;
// dst = (e * inv - l) * d_by_nr, d_by_nr = grad[0] / (float) nr.
__host__ __device__ __forceinline__ float ce_back_value(float e, float inv, float l, float d_by_nr) {
    return pool_mul(pool_add(pool_mul(e, inv), -l), d_by_nr);
}

// --------------------------------------------------------------------------------------------- REPEAT_BACK
// dst (k0, k1, k2, k3) = the sum, from +0, of src (i0 ne0 + k0, i1 ne1 + k1, i2 ne2 + k2, i3 ne3 + k3) over the repeats in ggml-cpu's loop
// order: i3, then i2, then i1, then i0 (ggml-cpu.c:6058-6072 adds one dst row per innermost step, so every element sees that order).
struct repeat_back_geom {
    int64_t ne[4];              // dst extents
    int64_t nr[4];              // repeats per dim: src ne / dst ne
    int64_t snb[4], dnb[4];     // strides, bytes
};

inline repeat_back_geom repeat_back_geometry(const ggml_b200_tensor & src, const ggml_b200_tensor & dst) {
    repeat_back_geom g;
    for (int i = 0; i < 4; ++i) {
        g.ne[i] = dst.ne[i]; g.nr[i] = dst.ne[i] ? src.ne[i] / dst.ne[i] : 0;
        g.snb[i] = (int64_t)src.nb[i]; g.dnb[i] = (int64_t)dst.nb[i];
    }
    return g;
}

// dst element e (linear, in dst's logical order): returns its byte offset in dst, and its value in *out
__host__ __device__ __forceinline__ int64_t repeat_back_value(const repeat_back_geom & g, const uint8_t * src, int64_t e, float * out) {
    const int64_t k0 = e % g.ne[0], q0 = e / g.ne[0], k1 = q0 % g.ne[1], q1 = q0 / g.ne[1], k2 = q1 % g.ne[2], k3 = q1 / g.ne[2];
    float acc = 0.0f;
    for (int64_t i3 = 0; i3 < g.nr[3]; ++i3)
        for (int64_t i2 = 0; i2 < g.nr[2]; ++i2)
            for (int64_t i1 = 0; i1 < g.nr[1]; ++i1) {
                const uint8_t * row = src + (i3 * g.ne[3] + k3) * g.snb[3] + (i2 * g.ne[2] + k2) * g.snb[2] + (i1 * g.ne[1] + k1) * g.snb[1];
                for (int64_t i0 = 0; i0 < g.nr[0]; ++i0) acc = pool_add(acc, *(const float *)(row + (i0 * g.ne[0] + k0) * g.snb[0]));
            }
    *out = acc;
    return k0 * g.dnb[0] + k1 * g.dnb[1] + k2 * g.dnb[2] + k3 * g.dnb[3];
}

// --------------------------------------------------------------------------------------------- STEP
__host__ __device__ __forceinline__ float step_value(float x) { return x > 0.0f ? 1.0f : 0.0f; }

// the reductions to a scalar (CROSS_ENTROPY_LOSS, SUM, COUNT_EQUAL) run in one CTA of RED_THREADS threads, in a fixed order, without atomics
enum { RED_THREADS = 1024 };

} // namespace b200
