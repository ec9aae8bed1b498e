// b200_sam.cuh — the per-element logic of the ops of a Segment-Anything-style image encoder and mask decoder, as ggml-cpu computes them
// (src/ggml-cpu/ggml-cpu.c): WIN_PART :11541-11582, WIN_UNPART :11604-11640, GET_REL_POS :11737-11760, ADD_REL_POS :11784-11842,
// CONV_TRANSPOSE_2D :10140-10230.  __host__ __device__, so that tests/hostemu compiles the same code for the CPU.
//
// The four data ops move raw 4- or 2-byte words: their results are bit-identical to ggml-cpu, NaN payloads and -0 included.  ADD_REL_POS
// takes its two adds in ggml-cpu's order (below), each correctly rounded: bit-identical.  CONV_TRANSPOSE_2D rounds the input to fp16 as
// ggml-cpu does and adds its taps in ggml-cpu's order; only the order of the Cin terms inside one tap's dot differs from ggml-cpu's SIMD sum.
//
// Row and plane indices are 32-bit: the checks (b200_op_checks.h) bound every row count by INT32_MAX.
#pragma once

#include "../../include/ggml-b200.h"
#include "b200_pool.cuh"

#include <cstdint>

namespace b200 {

// --------------------------------------------------------------------------------------------- WIN_PART
// src f32 [C, W0, H0, 1] packed -> dst f32 [C, w, w, npx npy] packed.  dst row r = (i1, i2, i3) = (r % w, (r / w) % w, r / (w w)) is the
// window i3 = py npx + px, pixel (i1, i2) of it: src row (py w + i2) W0 + (px w + i1), or zeros where the window runs past the image.
struct win_geom {
    int32_t w, npx;                 // window size, windows per image row
    int32_t W0, H0;                 // image extents (WIN_PART's src, WIN_UNPART's dst)
};

// the src row of WIN_PART's dst row r, -1 for a row of zeros
__host__ __device__ __forceinline__ int32_t win_part_src_row(const win_geom & g, uint32_t r) {
    const uint32_t w = (uint32_t)g.w, i1 = r % w, q = r / w, i2 = q % w, i3 = q / w;
    const uint32_t py = i3 / (uint32_t)g.npx, px = i3 - py * (uint32_t)g.npx;
    const uint32_t x = px * w + i1, y = py * w + i2;
    return x < (uint32_t)g.W0 && y < (uint32_t)g.H0 ? (int32_t)(y * (uint32_t)g.W0 + x) : -1;
}

// --------------------------------------------------------------------------------------------- WIN_UNPART
// src f32 [C, w, w, np] packed -> dst f32 [C, W0, H0, 1] packed.  dst row r = (i1, i2) = (r % W0, r / W0) comes from window
// (i2 / w) npx + i1 / w, pixel (i1 % w, i2 % w), npx = ceil(W0 / w) (ggml-cpu derives it from W0 the same way).
__host__ __device__ __forceinline__ uint32_t win_unpart_src_row(const win_geom & g, uint32_t r) {
    const uint32_t w = (uint32_t)g.w, i1 = r % (uint32_t)g.W0, i2 = r / (uint32_t)g.W0;
    const uint32_t wy = i2 / w, wx = i1 / w;
    return ((wy * (uint32_t)g.npx + wx) * w + (i2 - wy * w)) * w + (i1 - wx * w);
}

// --------------------------------------------------------------------------------------------- GET_REL_POS
// src f16 [C, 2w - 1] packed rows -> dst f16 [C, w, w] packed: dst row r = (i1, i2) = (r % w, r / w) is src row (w - 1 - i1) + i2
__host__ __device__ __forceinline__ uint32_t get_rel_pos_src_row(uint32_t w, uint32_t r) {
    const uint32_t i2 = r / w, i1 = r - i2 * w;
    return (w - 1 - i1) + i2;
}

// --------------------------------------------------------------------------------------------- ADD_REL_POS
// src0 / dst f32 [L L, A B, P, 1] packed; pw = src1, ph = src2 f32 [L, A, B, P] packed.  Row r of dst (0 <= r < A B P) holds the
// attention of query r over the L x L keys; key c = kh L + kw gets ph[r, kh] and pw[r, kw].
//
// ggml-cpu's loop (ggml-cpu.c:11823-11840) visits i10 = 0 .. L-1 and, for each, adds ph[r, i10] to the keys (kh = i10, kw = j) and then
// pw[r, i10] to the keys (kh = j, kw = i10), j = 0 .. L-1.  Key (kh, kw) therefore receives ph at i10 = kh and pw at i10 = kw: ph first
// when kh < kw, pw first when kh > kw, and when kh == kw ph first (the two adds of the same i10, in that order).
__host__ __device__ __forceinline__ float add_rel_pos_value(float a, float pw, float ph, uint32_t kh, uint32_t kw) {
    return kh <= kw ? pool_add(pool_add(a, ph), pw) : pool_add(pool_add(a, pw), ph);
}

// --------------------------------------------------------------------------------------------- CONV_TRANSPOSE_2D
// kernel f16 [Kw, Kh, Cout, Cin] (planes of Kw x Kh packed, any plane strides), input f32 [W, H, Cin, 1] (elements packed along dim 0,
// any row / channel strides) -> dst f32 [(W-1) s + Kw, (H-1) s + Kh, Cout, 1] packed.  Output (ox, oy, co) is the sum, from +0.0, over
// the input pixels (ix, iy) with kx = ox - ix s in [0, Kw) and ky = oy - iy s in [0, Kh), in ascending iy then ascending ix (the order in
// which ggml-cpu adds them into its zeroed dst), of one tap: dot = sum over ci ascending of fp16(input[ix, iy, ci]) x kernel[kx, ky, co, ci],
// each fp16 x fp16 product exact in f32 and each add rounded.
struct ct2d_geom {
    int32_t W, H, Cin, Kw, Kh, Cout, OW, OH, s;
    int64_t knb2, knb3;             // kernel plane strides (Cout, Cin), bytes
    int64_t xnb1, xnb2;             // input row / channel strides, bytes
};

inline ct2d_geom ct2d_geometry(const ggml_b200_tensor & kernel, const ggml_b200_tensor & input, const ggml_b200_tensor & dst, int32_t s) {
    ct2d_geom g;
    g.Kw = (int32_t)kernel.ne[0]; g.Kh = (int32_t)kernel.ne[1]; g.Cout = (int32_t)kernel.ne[2]; g.Cin = (int32_t)kernel.ne[3];
    g.W = (int32_t)input.ne[0]; g.H = (int32_t)input.ne[1];
    g.OW = (int32_t)dst.ne[0]; g.OH = (int32_t)dst.ne[1]; g.s = s;
    g.knb2 = (int64_t)kernel.nb[2]; g.knb3 = (int64_t)kernel.nb[3];
    g.xnb1 = (int64_t)input.nb[1]; g.xnb2 = (int64_t)input.nb[2];
    return g;
}

// the input element (ix, iy, ci) rounded to fp16 (as ggml-cpu's GGML_FP32_TO_FP16 rounds: to nearest even), as f32
__host__ __device__ __forceinline__ float ct2d_input(const ct2d_geom & g, const uint8_t * x, int32_t ix, int32_t iy, int32_t ci) {
    return __half2float(__float2half_rn(*(const float *)(x + (int64_t)ci * g.xnb2 + (int64_t)iy * g.xnb1 + (int64_t)ix * 4)));
}

// the kernel element (kx, ky, co, ci) as f32
__host__ __device__ __forceinline__ float ct2d_kernel(const ct2d_geom & g, const uint8_t * k, int32_t kx, int32_t ky, int32_t co, int32_t ci) {
    return __half2float(*(const __half *)(k + (int64_t)ci * g.knb3 + (int64_t)co * g.knb2 + ((int64_t)ky * g.Kw + kx) * 2));
}

// one tap's dot over Cin: ascending ci, products exact in f32, each add rounded (a fused multiply-add gives the same bits)
__host__ __device__ __forceinline__ float ct2d_dot_step(float dot, float x, float k) { return pool_add(dot, pool_mul(x, k)); }

// output (ox, oy, co) as the device kernel computes it, one output at a time (the host test's path; ops.cu's ct2d_kernel computes the same
// sums tiled, with the same order of taps and of ci)
inline float ct2d_value(const ct2d_geom & g, const uint8_t * k, const uint8_t * x, int32_t ox, int32_t oy, int32_t co) {
    float out = 0.0f;
    for (int32_t iy = 0; iy < g.H; ++iy) {
        const int32_t ky = oy - iy * g.s;
        if (ky < 0 || ky >= g.Kh) continue;
        for (int32_t ix = 0; ix < g.W; ++ix) {
            const int32_t kx = ox - ix * g.s;
            if (kx < 0 || kx >= g.Kw) continue;
            float dot = 0.0f;
            for (int32_t ci = 0; ci < g.Cin; ++ci) dot = ct2d_dot_step(dot, ct2d_input(g, x, ix, iy, ci), ct2d_kernel(g, k, kx, ky, co, ci));
            out = pool_add(out, dot);
        }
    }
    return out;
}

// the device tiling: a CTA owns CT2D_TQX x CT2D_TQY outputs of one stride phase (ox % s, oy % s) and CT2D_CO output channels; its 256
// threads are CT2D_CO / CT2D_COT channel groups of CT2D_TQX CT2D_TQY pixels, each thread one pixel x CT2D_COT channels.  Per tap and
// chunk of CT2D_CI input channels, the CTA stages the fp16-rounded input tile and the kernel slice in shared memory.
enum { CT2D_TQX = 32, CT2D_TQY = 2, CT2D_CO = 32, CT2D_COT = 8, CT2D_CI = 32, CT2D_THREADS = 256 };

} // namespace b200
