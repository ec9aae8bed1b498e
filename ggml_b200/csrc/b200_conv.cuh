// b200_conv.cuh — the per-element logic of GGML_OP_IM2COL (the lowering of ggml_conv_1d / ggml_conv_2d to a mat-mul), as
// ggml_compute_forward_im2col_f32 / _f16 compute it (src/ggml-cpu/ggml-cpu.c:9875-10041).  __host__ __device__, so that tests/hostemu
// compiles the same code for the CPU.
//
// dst is [IC KH KW, OW, OH, N] (1-D: [IC KW, OW, N, 1]) and written as if packed, element e in ggml's order.  Element (c, iow, ioh, in)
// with c = iic KH KW + ikh KW + ikw is src1 at column iow s0 + ikw d0 - p0, row ioh s1 + ikh d1 - p1 of channel iic of image in, or 0
// where that position lies in the padding.  Like the CPU, a channel's rows are read as packed (row iih at iih * IW elements, whatever
// src1's row stride), and the image / channel offsets are the strides the CPU keeps (nb3 / nb2 in 2-D, nb2 / nb1 in 1-D).  Each value is
// copied, or rounded once to fp16 by __float2half_rn, which rounds to nearest even as F16C does: both dst types are bit-identical to the CPU.
#pragma once

#include "../../include/ggml-b200.h"

#include <cstdint>

namespace b200 {

struct im2col_geom {
    int64_t N, IC, IH, IW, KH, KW, OH, OW;
    int64_t ofs0, ofs1;                  // src1 byte offsets of an image and of a channel
    int64_t s0, s1, p0, p1, d0, d1;
};

// the geometry as the CPU derives it from src0 (the kernel: only its extents), src1 (the input) and dst
inline im2col_geom im2col_geometry(const ggml_b200_tensor & src0, const ggml_b200_tensor & src1, const ggml_b200_tensor & dst,
                                   const ggml_b200_im2col_params & c) {
    const bool is_2D = c.is_2D == 1;
    im2col_geom g;
    g.N  = is_2D ? src1.ne[3] : src1.ne[2];
    g.IC = is_2D ? src1.ne[2] : src1.ne[1];
    g.IH = is_2D ? src1.ne[1] : 1;
    g.IW = src1.ne[0];
    g.KH = is_2D ? src0.ne[1] : 1;
    g.KW = src0.ne[0];
    g.OH = is_2D ? dst.ne[2] : 1;
    g.OW = dst.ne[1];
    g.ofs0 = (int64_t)(is_2D ? src1.nb[3] : src1.nb[2]);
    g.ofs1 = (int64_t)(is_2D ? src1.nb[2] : src1.nb[1]);
    g.s0 = c.s0; g.s1 = c.s1; g.p0 = c.p0; g.p1 = c.p1; g.d0 = c.d0; g.d1 = c.d1;
    return g;
}

// dst element e (0 <= e < N OH OW IC KH KW) read from src1's bytes
__host__ __device__ __forceinline__ float im2col_value(const im2col_geom & g, const uint8_t * src1, int64_t e) {
    const int64_t ckk = g.IC * g.KH * g.KW;
    const int64_t c = e % ckk, row = e / ckk;
    const int64_t iic = c / (g.KH * g.KW), ikh = (c / g.KW) % g.KH, ikw = c % g.KW;
    const int64_t iow = row % g.OW, ioh = (row / g.OW) % g.OH, in = row / (g.OW * g.OH);
    const int64_t iiw = iow * g.s0 + ikw * g.d0 - g.p0;
    const int64_t iih = ioh * g.s1 + ikh * g.d1 - g.p1;
    if (iih < 0 || iih >= g.IH || iiw < 0 || iiw >= g.IW) return 0.0f;
    return *(const float *)(src1 + in * g.ofs0 + iic * g.ofs1 + (iih * g.IW + iiw) * 4);
}

} // namespace b200
