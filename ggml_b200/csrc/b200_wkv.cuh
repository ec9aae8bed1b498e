// b200_wkv.cuh — the per-element math of GGML_OP_RWKV_WKV6 (the RWKV-6 time-mix recurrence) and GGML_OP_GATED_LINEAR_ATTN (its gated form,
// as RWKV6-Qwen2 models use it), as ggml_compute_forward_rwkv_wkv6_f32 / ggml_compute_forward_gla_f32 compute them
// (src/ggml-cpu/ggml-cpu.c:11865-12235).  __host__ __device__, so that tests/hostemu compiles the same code for the CPU.
//
// For one token of one head, with state[i][j] the head's S x S state (row i = key index, column j = value index):
//   WKV6: kv = v[j] k[i];  y[j] += (kv tf[i] + state[i][j]) r[i];   state[i][j] = state[i][j] td[i] + kv
//   GLA:  kv = v[j] k[i];  temp = state[i][j] g[i] + kv;  y[j] += temp (q[i] scale);  state[i][j] = temp
// with y[j] summed over i in ascending order from 0.
//
// Parity with ggml-cpu: its vector path (every column when S is a multiple of the build's vector width: 8 with AVX2, 16 with AVX-512)
// multiplies kv, then fuses each multiply-add into one FMA, and rounds q[i] * scale on its own.  The expressions below spell exactly that
// rounding out with explicit fused / unfused operations, so the result is bit-identical there on both host and device (nvcc would
// otherwise contract on its own).  For other head sizes ggml-cpu computes its tail columns (j beyond the last whole vector) unfused,
// because the reference is built -std=c11 and gcc does not contract there; which columns that is depends on the CPU build.  This code
// does not copy that build detail: those columns agree to f32 round-off, the others bit for bit.
#pragma once

#include <cmath>
#include <cstdint>

// on the device the row loops are unrolled so that the state loads of several rows are in flight at once (the sums stay in order)
#ifdef __CUDA_ARCH__
#define B200_WKV_UNROLL _Pragma("unroll 8")
#else
#define B200_WKV_UNROLL
#endif

namespace b200 {

__host__ __device__ __forceinline__ float wkv_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ float wkv_fma(float a, float b, float c) {
#ifdef __CUDA_ARCH__
    return __fmaf_rn(a, b, c);
#else
    return std::fma(a, b, c);
#endif
}

// WKV6, one token, column j of one head: returns y[j] and writes the column's new state.  k, r, tf, td point at the head's S values of
// this token (tf: of the head); prev[i * stride] / st[i * stride] is state[i][j] before / after the token (st may be prev).
__host__ __device__ __forceinline__ float wkv6_column(const float * k, const float * r, const float * tf, const float * td, float v,
                                                      const float * prev, float * st, int64_t stride, int64_t S) {
    float y = 0.0f;
    B200_WKV_UNROLL
    for (int64_t i = 0; i < S; ++i) {
        const float p = prev[i * stride];
        const float kv = wkv_mul(v, k[i]);
        y = wkv_fma(wkv_fma(kv, tf[i], p), r[i], y);
        st[i * stride] = wkv_fma(p, td[i], kv);
    }
    return y;
}

// GLA, one token, column j of one head; qs[i] = q[i] * scale, rounded (gla_scaled_q).  The other arguments as for wkv6_column.
__host__ __device__ __forceinline__ float gla_scaled_q(float q, float scale) { return wkv_mul(q, scale); }
__host__ __device__ __forceinline__ float gla_column(const float * k, const float * qs, const float * g, float v,
                                                     const float * prev, float * st, int64_t stride, int64_t S) {
    float y = 0.0f;
    B200_WKV_UNROLL
    for (int64_t i = 0; i < S; ++i) {
        const float temp = wkv_fma(prev[i * stride], g[i], wkv_mul(v, k[i]));
        y = wkv_fma(temp, qs[i], y);
        st[i * stride] = temp;
    }
    return y;
}

} // namespace b200
