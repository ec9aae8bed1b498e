// b200_rope.cuh — the per-pair math of GGML_OP_ROPE (forward), as ggml_compute_forward_rope_f32 / _f16 compute it
// (src/ggml-cpu/ggml-cpu.c:9157-9438).  __host__ __device__, so that tests/hostemu compiles the same code for the CPU.
//
// Parity with ggml-cpu: every per-op constant (theta_scale, the YaRN corr dims, the magnitude mscale) is computed on the host with
// the CPU's own expressions and passed in; theta of pair j is rebuilt by the same sequential product theta *= theta_scale as
// ggml_rope_cache_init / ggml_mrope_cache_init (never powf(theta_scale, j)); every multiply-add is rounded per operation as the
// CPU build (-ffp-contract=off) does.  What remains different is the device sinf / cosf versus glibc's: a few ulp.
#pragma once

#include <cstdint>

#include "b200_op_checks.h"     // the modes, ROPE_MAX_CACHE and rope_n_cache

namespace b200 {

// the per-op constants are the ABI struct itself: the launcher hands the caller's ggml_b200_rope_params to the kernel as it is
using rope_consts = ggml_b200_rope_params;

// separately rounded multiply / add / subtract (no FMA contraction on the device)
__host__ __device__ __forceinline__ float rp_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ float rp_add(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ float rp_sub(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}

// theta of pair j (cache slot i0 = 2j) before the freq-factor division; p[0..3]: the position streams (only p[0] outside MROPE)
__host__ __device__ inline float rope_theta(const rope_consts & c, const float * p, int j) {
    if (!(c.mode & ROPE_MROPE)) {
        float t = p[0];
        for (int k = 0; k < j; ++k) t = rp_mul(t, c.theta_scale);
        return t;
    }
    // MROPE: four streams advanced together; sector k % sect_dims picks the stream; VISION restarts a stream at its section's start
    const int s0 = c.sections[0], sec_w = s0 + c.sections[1], sec_e = sec_w + c.sections[2], sect_dims = sec_e + c.sections[3];
    const bool indep = c.mode == ROPE_VISION;
    float tt = p[0], th = p[1], tw = p[2], te = p[3];
    int sector = 0;
    for (int k = 0;; ++k) {
        if (indep) {
            if (sector == 0) tt = p[0];
            else if (sector == s0) th = p[1];
            else if (sector == sec_w) tw = p[2];
            else if (sector == sec_e) te = p[3];
        }
        if (k == j) {
            if (sector >= s0 && sector < sec_w) return th;
            if (sector >= sec_w && sector < sec_e) return tw;
            if (sector >= sec_e) return te;
            return tt;
        }
        tt = rp_mul(tt, c.theta_scale); th = rp_mul(th, c.theta_scale);
        tw = rp_mul(tw, c.theta_scale); te = rp_mul(te, c.theta_scale);
        if (++sector == sect_dims) sector = 0;
    }
}

// cos / sin (times mscale) of pair j with YaRN: theta_extrap = theta / ff, interpolated by freq_scale, ramped between the corr dims
__host__ __device__ inline void rope_cos_sin(const rope_consts & c, float theta, float ff, int j, float & cs, float & sn) {
    const float extrap = theta / ff;
    const float interp = rp_mul(c.freq_scale, extrap);
    float t = interp;
    if (c.ext_factor != 0.0f) {
        const float span = rp_sub(c.corr_dims[1], c.corr_dims[0]);
        const float y = rp_sub((float)j, c.corr_dims[0]) / (0.001f > span ? 0.001f : span);
        const float lo = 0.0f > y ? 0.0f : y;
        const float ramp = rp_sub(1.0f, 1.0f < lo ? 1.0f : lo);
        const float mix = rp_mul(ramp, c.ext_factor);
        t = rp_add(rp_mul(interp, rp_sub(1.0f, mix)), rp_mul(extrap, mix));
    }
    cs = rp_mul(cosf(t), c.mscale);
    sn = rp_mul(sinf(t), c.mscale);
}

// item q of a row (0 <= q < ne0/2): the two element indices it owns, and the cache slot it rotates by (-1: copied unchanged)
__host__ __device__ __forceinline__ int rope_item(const rope_consts & c, int64_t q, int64_t & e0, int64_t & e1) {
    const int64_t half = c.n_dims / 2;
    if (c.mode == ROPE_VISION) { e0 = q; e1 = q + c.n_dims; return (int)q; }
    if (q >= half) { e0 = 2 * q; e1 = 2 * q + 1; return -1; }              // the tail beyond n_dims
    if (c.mode == ROPE_NORM) { e0 = 2 * q; e1 = 2 * q + 1; }                  // adjacent pairs
    else { e0 = q; e1 = q + half; }                                            // NEOX / MROPE: i, i + n_dims/2
    return (int)q;
}

__host__ __device__ __forceinline__ void rope_rotate(float x0, float x1, float cs, float sn, float & y0, float & y1) {
    y0 = rp_sub(rp_mul(x0, cs), rp_mul(x1, sn));
    y1 = rp_add(rp_mul(x0, sn), rp_mul(x1, cs));
}

} // namespace b200
