// b200_ssm.cuh — the per-element math of GGML_OP_SSM_CONV and GGML_OP_SSM_SCAN (the Mamba-1 layer), as ggml_compute_forward_ssm_conv_f32 /
// ggml_compute_forward_ssm_scan_f32 compute it (src/ggml-cpu/ggml-cpu.c:11379-11537).  __host__ __device__, so that tests/hostemu compiles
// the same code for the CPU.
//
// Parity with ggml-cpu: every multiply and every add is rounded separately (the CPU build, -std=c11, does not contract to FMA; nvcc would),
// and the sums run in the CPU's order: ascending i0 from 0.0f.  SSM_CONV is therefore bit-identical to ggml-cpu.  SSM_SCAN differs only
// where the device expf / log1pf differ from glibc's (a few ulp); compiled for the host it is bit-identical.
#pragma once

#include <cmath>
#include <cstdint>

namespace b200 {

__host__ __device__ __forceinline__ float ssm_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ float ssm_add(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

// SSM_CONV, one output: the dot product of the window s[0 .. nc) of a conv_x row with the row c[0 .. nc) of the conv1d weight
__host__ __device__ __forceinline__ float ssm_conv_dot(const float * s, const float * c, int64_t nc) {
    float sumf = 0.0f;
    for (int64_t i0 = 0; i0 < nc; ++i0) sumf = ssm_add(sumf, ssm_mul(s[i0], c[i0]));
    return sumf;
}

// softplus of the time step, with the CPU's cut-off: dt itself above 20
__host__ __device__ __forceinline__ float ssm_softplus(float dt) { return dt <= 20.0f ? log1pf(expf(dt)) : dt; }

// SSM_SCAN, one token of one row i1: state[i0] = s0[i0] * exp(dt_sp * A[i0]) + B[i0] * (x * dt_sp) for i0 < nc, written to s (s may be s0);
// returns y = sum_i0 state[i0] * C[i0].  A, B, C point at the row's / token's d_state values (contiguous).
__host__ __device__ __forceinline__ float ssm_scan_token(const float * s0, float * s, const float * A, const float * B, const float * C, float x, float dt,
                                                        int64_t nc) {
    const float dt_sp = ssm_softplus(dt);
    const float x_dt = ssm_mul(x, dt_sp);
    float sumf = 0.0f;
    for (int64_t i0 = 0; i0 < nc; ++i0) {
        const float state = ssm_add(ssm_mul(s0[i0], expf(ssm_mul(dt_sp, A[i0]))), ssm_mul(B[i0], x_dt));
        sumf = ssm_add(sumf, ssm_mul(state, C[i0]));
        s[i0] = state;
    }
    return sumf;
}

} // namespace b200
