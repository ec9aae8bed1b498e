// b200_pool.cuh — the per-element logic of the ops around the convolutions of a YOLO-style network, as ggml-cpu computes them
// (src/ggml-cpu/ggml-cpu.c): POOL_2D :10305-10377, UPSCALE :10503-10540, LEAKY_RELU :6689-6717 (expression :1741), REPEAT :5901-6015.
// __host__ __device__, so that tests/hostemu compiles the same code for the CPU.
//
// Every result is bit-identical to ggml-cpu: each arithmetic step is one correctly rounded IEEE operation (pool_add / pool_mul / pool_div
// below), taken in the CPU's order, and REPEAT moves raw words.
#pragma once

#include "../../include/ggml-b200.h"

#include <cfloat>
#include <cstdint>

namespace b200 {

// one correctly rounded IEEE operation each: __fadd_rn / __fmul_rn / __fdiv_rn on the device (never contracted or approximated), the
// plain operator on the host (tests/hostemu builds with -ffp-contract=off)
__host__ __device__ __forceinline__ float pool_add(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ float pool_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ float pool_div(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}

enum { POOL_MAX = 0, POOL_AVG = 1, POOL_COUNT = 2 };     // enum ggml_op_pool

// --------------------------------------------------------------------------------------------- POOL_2D
// dst [OW, OH, C, N] f32, written packed; src f32 [IW, IH, C, N], elements packed along dim 0, rows at nb1, channels at nb2, images at nb3.
// The extents come from dst, never from the parameters: ggml_pool_2d derives them from float paddings and stores the paddings truncated.
struct pool2d_geom {
    int64_t IW, IH, OW, OH, C;
    int64_t nb1, nb2, nb3;
    int32_t op, k0, k1, s0, s1, p0, p1;
};

inline pool2d_geom pool2d_geometry(const ggml_b200_tensor & src, const ggml_b200_tensor & dst, const ggml_b200_pool_params & p) {
    pool2d_geom g;
    g.IW = src.ne[0]; g.IH = src.ne[1]; g.OW = dst.ne[0]; g.OH = dst.ne[1]; g.C = src.ne[2];
    g.nb1 = (int64_t)src.nb[1]; g.nb2 = (int64_t)src.nb[2]; g.nb3 = (int64_t)src.nb[3];
    g.op = p.op; g.k0 = p.k0; g.k1 = p.k1; g.s0 = p.s0; g.s1 = p.s1; g.p0 = p.p0; g.p1 = p.p1;
    return g;
}

// dst element e (0 <= e < OW OH C N).  MAX starts at -FLT_MAX and takes a tap only when it is greater: NaN taps are skipped, a window
// with nothing greater gives -FLT_MAX, and of equal taps (+0 / -0) the first stays.  AVG adds the in-range taps to 0 in ky-major, kx-minor
// order and divides once by k0 k1, so taps in the padding count in the divisor.  The window origin is int arithmetic, as on the CPU.
__host__ __device__ __forceinline__ float pool2d_value(const pool2d_geom & g, const uint8_t * src, int64_t e) {
    const int64_t ox = e % g.OW, oy = (e / g.OW) % g.OH, c = (e / (g.OW * g.OH)) % g.C, n = e / (g.OW * g.OH * g.C);
    const uint8_t * plane = src + c * g.nb2 + n * g.nb3;
    const int ix = -g.p0 + (int)ox * g.s0, iy = -g.p1 + (int)oy * g.s1;
    float out = g.op == POOL_AVG ? 0.0f : -FLT_MAX;
    for (int ky = 0; ky < g.k1; ++ky) {
        if (iy + ky < 0 || iy + ky >= g.IH) continue;
        const float * row = (const float *)(plane + g.nb1 * (iy + ky));
        for (int kx = 0; kx < g.k0; ++kx) {
            const int j = ix + kx;
            if (j < 0 || j >= g.IW) continue;
            const float v = row[j];
            if (g.op == POOL_AVG) out = pool_add(out, v);
            else if (v > out) out = v;
        }
    }
    return g.op == POOL_AVG ? pool_div(out, (float)(g.k0 * g.k1)) : out;
}

// --------------------------------------------------------------------------------------------- UPSCALE (nearest)
// dst [ne0 .. ne3] element (i0, i1, i2, i3) is src element (i0 / sf0, ...) truncated, sf_i = (float)ne_i / src ne_i, all in float as the
// CPU computes them (the host evaluates the factors; the division per element is pool_div).  Any src and dst strides.
struct upscale_geom {
    int64_t ne[4];                  // dst extents
    int64_t snb[4], dnb[4];         // byte strides of src and dst
    float sf[4];
};

inline upscale_geom upscale_geometry(const ggml_b200_tensor & src, const ggml_b200_tensor & dst) {
    upscale_geom g;
    for (int i = 0; i < 4; ++i) {
        g.ne[i] = dst.ne[i]; g.snb[i] = (int64_t)src.nb[i]; g.dnb[i] = (int64_t)dst.nb[i];
        g.sf[i] = (float)dst.ne[i] / src.ne[i];
    }
    return g;
}

// the byte offsets in src (returned) and dst (dofs) of dst element e, in dst's logical order
__host__ __device__ __forceinline__ int64_t upscale_offsets(const upscale_geom & g, int64_t e, int64_t & dofs) {
    const int64_t i0 = e % g.ne[0], i1 = (e / g.ne[0]) % g.ne[1], i2 = (e / (g.ne[0] * g.ne[1])) % g.ne[2], i3 = e / (g.ne[0] * g.ne[1] * g.ne[2]);
    const int64_t s0 = (int64_t)pool_div((float)i0, g.sf[0]), s1 = (int64_t)pool_div((float)i1, g.sf[1]);
    const int64_t s2 = (int64_t)pool_div((float)i2, g.sf[2]), s3 = (int64_t)pool_div((float)i3, g.sf[3]);
    dofs = i0 * g.dnb[0] + i1 * g.dnb[1] + i2 * g.dnb[2] + i3 * g.dnb[3];
    return s0 * g.snb[0] + s1 * g.snb[1] + s2 * g.snb[2] + s3 * g.snb[3];
}

// --------------------------------------------------------------------------------------------- LEAKY_RELU
// ((x > 0) ? x : 0) + slope ((x < 0) ? x : 0): NaN and -0 become +0
__host__ __device__ __forceinline__ float leaky_relu_value(float x, float slope) {
    return pool_add(x > 0.0f ? x : 0.0f, pool_mul(slope, x < 0.0f ? x : 0.0f));
}

// --------------------------------------------------------------------------------------------- REPEAT
// dst element (i0, i1, i2, i3) is src element (i0 % ne00, i1 % ne01, ...) (whole repeats only).  Returns the byte offsets in src (returned)
// and dst (dofs) of dst element e, in dst's logical order; the caller moves one element-sized word, so every bit pattern survives.
struct repeat_geom {
    int64_t ne[4], sne[4];          // dst and src extents
    int64_t snb[4], dnb[4];
};

inline repeat_geom repeat_geometry(const ggml_b200_tensor & src, const ggml_b200_tensor & dst) {
    repeat_geom g;
    for (int i = 0; i < 4; ++i) { g.ne[i] = dst.ne[i]; g.sne[i] = src.ne[i]; g.snb[i] = (int64_t)src.nb[i]; g.dnb[i] = (int64_t)dst.nb[i]; }
    return g;
}

__host__ __device__ __forceinline__ int64_t repeat_offsets(const repeat_geom & g, int64_t e, int64_t & dofs) {
    const int64_t i0 = e % g.ne[0], i1 = (e / g.ne[0]) % g.ne[1], i2 = (e / (g.ne[0] * g.ne[1])) % g.ne[2], i3 = e / (g.ne[0] * g.ne[1] * g.ne[2]);
    dofs = i0 * g.dnb[0] + i1 * g.dnb[1] + i2 * g.dnb[2] + i3 * g.dnb[3];
    return (i0 % g.sne[0]) * g.snb[0] + (i1 % g.sne[1]) * g.snb[1] + (i2 % g.sne[2]) * g.snb[2] + (i3 % g.sne[3]) * g.snb[3];
}

} // namespace b200
