// b200_tc_dequant.cuh — per-thread operand preparation of the tensor-core GEMM (mmq_tc2.cu): raw-unit geometry of the packed W formats and
// the conversion of 64 weights of one row to fp16 in the SWIZZLE_128B K-major layout the wgmma descriptors read.  Pure per-thread code, split from the
// kernel file so that tests/hostemu can compile it for the host and check it against the oracle in the CPU-only suite.
#pragma once
#include "b200_quants.cuh"

namespace b200 {

// ----------------------------------------------------------------------------- W raw-unit geometry
// The TMA producer copies W in "raw units": for every row of the tile the packed bytes of UNIT_KSTEPS x 64 consecutive weights
// (2-D tensor map over the byte matrix [M][row_bytes]: coalesced whatever the block size).  RAW = bytes of the TMA box per row
// (multiple of 16), STRIDE_WORDS = distance between consecutive units of a row in 4-byte words, UNIT_WORDS = payload words.
// A TMA box must start on a 16-byte boundary of the row: Q8_0 units are 136 B apart, so the box of an odd unit starts
// ODD_BACK_WORDS (8 bytes) early and its payload sits 8 bytes into the box (hence 8-byte shared-memory loads for Q8_0).
// A dequantizer thread first copies its row's unit into registers and releases the shared-memory buffer at once, so the
// raw pipeline is effectively three units deep.
template <int T> struct tcfmt;
template <> struct tcfmt<T_Q4_0> { static constexpr int RAW = 144, STRIDE_WORDS = 36, UNIT_WORDS = 36, UNIT_KSTEPS = 4, ODD_BACK_WORDS = 0, LOAD_BYTES = 16; };   // 8 blocks of 18 B
template <> struct tcfmt<T_Q8_0> { static constexpr int RAW = 144, STRIDE_WORDS = 34, UNIT_WORDS = 34, UNIT_KSTEPS = 2, ODD_BACK_WORDS = 2, LOAD_BYTES = 8;  };   // 4 blocks of 34 B
template <> struct tcfmt<T_Q4_K> { static constexpr int RAW = 144, STRIDE_WORDS = 36, UNIT_WORDS = 36, UNIT_KSTEPS = 4, ODD_BACK_WORDS = 0, LOAD_BYTES = 16; };   // one superblock
template <> struct tcfmt<T_Q5_K> { static constexpr int RAW = 176, STRIDE_WORDS = 44, UNIT_WORDS = 44, UNIT_KSTEPS = 4, ODD_BACK_WORDS = 0, LOAD_BYTES = 16; };
// Q6_K: 210-byte superblocks, 2-byte aligned: the TMA box starts on the 16-byte boundary below the unit and carries up to 14 bytes of
// lead (RAW = 224, payload offset 210 u mod 16).
template <> struct tcfmt<T_Q6_K> { static constexpr int RAW = 224, STRIDE_WORDS = 0, UNIT_WORDS = 53, UNIT_KSTEPS = 4, ODD_BACK_WORDS = 0, LOAD_BYTES = 2, UNIT_BYTES = 210; };
// SURVEY §8f-2 formats (decoders host-verified, kernels checked by the GPU suite).  16-byte-multiple units are loaded like Q4_0; the others
// (LOAD_BYTES = 2) use the variable-lead box: RAW = UNIT_BYTES + largest lead, rounded up to 16.
template <> struct tcfmt<T_Q4_1>   { static constexpr int RAW = 160, STRIDE_WORDS = 40, UNIT_WORDS = 40, UNIT_KSTEPS = 4, ODD_BACK_WORDS = 0, LOAD_BYTES = 16; };
template <> struct tcfmt<T_Q5_0>   { static constexpr int RAW = 176, STRIDE_WORDS = 44, UNIT_WORDS = 44, UNIT_KSTEPS = 4, ODD_BACK_WORDS = 0, LOAD_BYTES = 16; };
template <> struct tcfmt<T_Q5_1>   { static constexpr int RAW = 192, STRIDE_WORDS = 48, UNIT_WORDS = 48, UNIT_KSTEPS = 4, ODD_BACK_WORDS = 0, LOAD_BYTES = 16; };
template <> struct tcfmt<T_IQ4_NL> { static constexpr int RAW = 144, STRIDE_WORDS = 36, UNIT_WORDS = 36, UNIT_KSTEPS = 4, ODD_BACK_WORDS = 0, LOAD_BYTES = 16; };
template <> struct tcfmt<T_Q2_K>   { static constexpr int RAW = 96,  STRIDE_WORDS = 0,  UNIT_WORDS = 21, UNIT_KSTEPS = 4, ODD_BACK_WORDS = 0, LOAD_BYTES = 2, UNIT_BYTES = 84;  };
template <> struct tcfmt<T_Q3_K>   { static constexpr int RAW = 128, STRIDE_WORDS = 0,  UNIT_WORDS = 28, UNIT_KSTEPS = 4, ODD_BACK_WORDS = 0, LOAD_BYTES = 2, UNIT_BYTES = 110; };
template <> struct tcfmt<T_IQ4_XS> { static constexpr int RAW = 144, STRIDE_WORDS = 0,  UNIT_WORDS = 34, UNIT_KSTEPS = 4, ODD_BACK_WORDS = 0, LOAD_BYTES = 2, UNIT_BYTES = 136; };

template <int T> __device__ __forceinline__ void tc_load_unit(const uint8_t * g, uint32_t (&u)[tcfmt<T>::UNIT_WORDS]) {   // g: shared memory
    if constexpr (tcfmt<T>::LOAD_BYTES == 2) {
        load_words_a2<tcfmt<T>::UNIT_WORDS>(g, u);            // 2-byte aligned unit: aligned words + funnel shift
    } else if constexpr (tcfmt<T>::LOAD_BYTES == 16) {
#pragma unroll
        for (int i = 0; i < tcfmt<T>::UNIT_WORDS / 4; ++i) { const uint4 v = *((const uint4 *)g + i); u[4 * i] = v.x; u[4 * i + 1] = v.y; u[4 * i + 2] = v.z; u[4 * i + 3] = v.w; }
    } else {
#pragma unroll
        for (int i = 0; i < tcfmt<T>::UNIT_WORDS / 2; ++i) { const uint2 v = *((const uint2 *)g + i); u[2 * i] = v.x; u[2 * i + 1] = v.y; }
    }
}

// ---- integer codes -> fp16 without any int->float conversion: byte b under the exponent byte 0x64 is the half 1024 + b
// (ulp = 1 in [1024, 2048)), so "subtract the bias, multiply by the block scale" is two packed-half instructions per two weights.
__device__ __forceinline__ __half2 u2h(uint32_t u) { return *reinterpret_cast<__half2 *>(&u); }
__device__ __forceinline__ uint32_t h2u(__half2 h) { return *reinterpret_cast<uint32_t *>(&h); }
__device__ __forceinline__ __half2 bytes01_h2(uint32_t w) { return u2h(__byte_perm(w, 0x64646464u, 0x5140)); }   // (1024 + b0, 1024 + b1)
__device__ __forceinline__ __half2 bytes23_h2(uint32_t w) { return u2h(__byte_perm(w, 0x64646464u, 0x5342)); }   // (1024 + b2, 1024 + b3)
// four codes (bytes of w, each < 256) -> (code - bias) * d, packed halves
__device__ __forceinline__ void codes4_scale(uint32_t w, __half2 bias, __half2 d, uint32_t & o0, uint32_t & o1) {
    o0 = h2u(__hmul2(__hsub2(bytes01_h2(w), bias), d));
    o1 = h2u(__hmul2(__hsub2(bytes23_h2(w), bias), d));
}
// four codes -> code * d + m  (K-quants: d = super-scale x 6-bit scale, m = -(super-min x 6-bit min))
__device__ __forceinline__ void codes4_affine(uint32_t w, __half2 d, __half2 m, uint32_t & o0, uint32_t & o1) {
    const __half2 k1024 = __float2half2_rn(1024.0f);
    o0 = h2u(__hfma2(__hsub2(bytes01_h2(w), k1024), d, m));
    o1 = h2u(__hfma2(__hsub2(bytes23_h2(w), k1024), d, m));
}

// dequantize the 64 weights of K-step KS (0 .. UNIT_KSTEPS-1) of the unit held in registers `u` to fp16:
// 8 chunks of 8 halves (16 bytes), chunk c = k 8c..8c+7, each stored as soon as it is computed to its SWIZZLE_128B position
// (chunk index XOR row % 8) in the row's 128-byte line of the A stage.  Every index below is a compile-time constant.
#define TC_OUT(idx, r) (*(uint4 *)(a_row + (((uint32_t)(idx) ^ sw) << 4)) = (r))
template <int T, int KS, int UW = tcfmt<T>::UNIT_WORDS> __device__ __forceinline__ void dq64(const uint32_t (&u)[UW], uint8_t * a_row, uint32_t sw) {   // UW deduced: the pair kernel's Q8_0 unit is 8 blocks wide
    if constexpr (T == T_Q8_0) {
        // blocks 2KS, 2KS+1 of the unit: block b starts at byte 34 b = word 8.5 b; block 2KS at word 17 KS
        constexpr int o = 17 * KS;
        const __half2 bias = __float2half2_rn(1152.0f);         // 1024 + 128: the int8 codes are offset to 0..255 first
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const uint32_t dbits = b == 0 ? (u[o] & 0xFFFF) : (u[o + 8] >> 16);
            const __half2 d = u2h(dbits | (dbits << 16));       // the block scale already is an fp16
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                uint32_t q0, q1;
                if (b == 0) { q0 = __funnelshift_r(u[o + 2 * c], u[o + 2 * c + 1], 16); q1 = __funnelshift_r(u[o + 2 * c + 1], u[o + 2 * c + 2], 16); }
                else        { q0 = u[o + 9 + 2 * c]; q1 = u[o + 10 + 2 * c]; }
                uint4 r;
                codes4_scale(q0 ^ 0x80808080u, bias, d, r.x, r.y);
                codes4_scale(q1 ^ 0x80808080u, bias, d, r.z, r.w);
                TC_OUT(4 * b + c, r);
            }
        }
    } else if constexpr (T == T_Q4_0) {
        // blocks 2KS, 2KS+1: 36 bytes at word 9 KS
        constexpr int o = 9 * KS;
        const __half2 bias = __float2half2_rn(1032.0f);         // 1024 + 8
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const uint32_t dbits = b == 0 ? (u[o] & 0xFFFF) : (u[o + 4] >> 16);
            const __half2 d = u2h(dbits | (dbits << 16));
            uint32_t q[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) q[i] = b == 0 ? __funnelshift_r(u[o + i], u[o + i + 1], 16) : u[o + 5 + i];
            // byte j of qs: low nibble -> element j, high nibble -> element j + 16
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int hi = c >> 1;                          // chunks 0,1: elements 0..15 (low nibbles); 2,3: 16..31 (high)
                const uint32_t qa = (q[2 * (c & 1)] >> (4 * hi)) & 0x0F0F0F0F, qb = (q[2 * (c & 1) + 1] >> (4 * hi)) & 0x0F0F0F0F;
                uint4 r;
                codes4_scale(qa, bias, d, r.x, r.y);
                codes4_scale(qb, bias, d, r.z, r.w);
                TC_OUT(4 * b + c, r);
            }
        }
    } else if constexpr (T == T_Q6_K) {
        // K-step KS = half h = KS / 2 of the superblock, nibble pp = KS % 2 of ql (positions 2 pp and 2 pp + 1 of the reference's
        // interleave, src/ggml-quants.c:1690-1719): element 64 KS + j -> position 2 pp + j / 32, l = j % 32;
        // code = nibble pp of ql[64 h + 32 (pos % 2) + l] | bits 2 pos.. of qh[32 h + l] << 4; value = d * scales[8 h + l / 16 + 2 pos] * (code - 32)
        constexpr int h = KS >> 1, pp = KS & 1;
        const float dd = h2f(u[52] & 0xFFFF);
        const __half2 bias = __float2half2_rn(1056.0f);          // 1024 + 32
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int pos = 2 * pp + (c >> 2), l0 = 8 * (c & 3);                 // eight consecutive l of one position
            const int sidx = 8 * h + (l0 >> 4) + 2 * pos;                        // int8 scale of this 16-group (bytes 192..207)
            const int sc = (int)(int8_t)((u[48 + (sidx >> 2)] >> (8 * (sidx & 3))) & 0xFF);
            const __half2 d = __float2half2_rn(dd * (float)sc);
            uint4 r;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const uint32_t ql = u[16 * h + 8 * (pos & 1) + (l0 >> 2) + half], qh = u[32 + 8 * h + (l0 >> 2) + half];
                const uint32_t code = ((ql >> (4 * pp)) & 0x0F0F0F0Fu) | (((qh >> (2 * pos)) & 0x03030303u) << 4);
                if (half == 0) codes4_scale(code, bias, d, r.x, r.y); else codes4_scale(code, bias, d, r.z, r.w);
            }
            TC_OUT(c, r);
        }
    } else if constexpr (T == T_Q4_1 || T == T_Q5_0 || T == T_Q5_1 || T == T_IQ4_NL) {
        // 32-element blocks 2KS, 2KS+1 of the unit; block layouts: Q4_1 d|m, qs[16] (5 words); Q5_0 d, qh, qs (22 B, 2-byte granular);
        // Q5_1 d|m, qh, qs (6 words); IQ4_NL d, qs (18 B)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            constexpr int dummy = 0; (void)dummy;
            const int blk = 2 * KS + b;
            uint32_t q[4], qh = 0, dbits, mbits = 0;
            if constexpr (T == T_Q4_1) {
                dbits = u[5 * blk] & 0xFFFF; mbits = u[5 * blk] >> 16;
#pragma unroll
                for (int i = 0; i < 4; ++i) q[i] = u[5 * blk + 1 + i];
            } else if constexpr (T == T_Q5_1) {
                dbits = u[6 * blk] & 0xFFFF; mbits = u[6 * blk] >> 16; qh = u[6 * blk + 1];
#pragma unroll
                for (int i = 0; i < 4; ++i) q[i] = u[6 * blk + 2 + i];
            } else if constexpr (T == T_Q5_0) {
                const int w0 = (22 * blk) / 4;                   // byte 22 blk: word-aligned for even blk, half-word shifted for odd blk
                if ((blk & 1) == 0) {
                    dbits = u[w0] & 0xFFFF; qh = __funnelshift_r(u[w0], u[w0 + 1], 16);
#pragma unroll
                    for (int i = 0; i < 4; ++i) q[i] = __funnelshift_r(u[w0 + 1 + i], u[w0 + 2 + i], 16);
                } else {
                    dbits = u[w0] >> 16; qh = u[w0 + 1];
#pragma unroll
                    for (int i = 0; i < 4; ++i) q[i] = u[w0 + 2 + i];
                }
            } else {                                             // IQ4_NL: as Q4_0
                const int w0 = (18 * blk) / 4;
                if ((blk & 1) == 0) {
                    dbits = u[w0] & 0xFFFF;
#pragma unroll
                    for (int i = 0; i < 4; ++i) q[i] = __funnelshift_r(u[w0 + i], u[w0 + i + 1], 16);
                } else {
                    dbits = u[w0] >> 16;
#pragma unroll
                    for (int i = 0; i < 4; ++i) q[i] = u[w0 + 1 + i];
                }
            }
            const __half2 d = u2h(dbits | (dbits << 16)), m = u2h(mbits | (mbits << 16));
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int hi = c >> 1;                           // chunks 0,1: elements 0..15 (low nibbles); 2,3: 16..31 (high nibbles)
                uint32_t qa = (q[2 * (c & 1)] >> (4 * hi)) & 0x0F0F0F0F, qb = (q[2 * (c & 1) + 1] >> (4 * hi)) & 0x0F0F0F0F;
                uint4 r;
                if constexpr (T == T_Q4_1) {
                    codes4_affine(qa, d, m, r.x, r.y); codes4_affine(qb, d, m, r.z, r.w);
                } else if constexpr (T == T_IQ4_NL) {
                    const __half2 bias = __float2half2_rn(1152.0f);   // codebook entries are int8: offset to 0..255 first
                    codes4_scale(iq4nl_lookup4(qa) ^ 0x80808080u, bias, d, r.x, r.y); codes4_scale(iq4nl_lookup4(qb) ^ 0x80808080u, bias, d, r.z, r.w);
                } else {
                    const int bit0 = 16 * hi + 8 * (c & 1);      // fifth bit of the chunk's first element
                    qa |= spread4_to_bit4(qh >> bit0); qb |= spread4_to_bit4(qh >> (bit0 + 4));
                    if constexpr (T == T_Q5_1) { codes4_affine(qa, d, m, r.x, r.y); codes4_affine(qb, d, m, r.z, r.w); }
                    else { const __half2 bias = __float2half2_rn(1040.0f); codes4_scale(qa, bias, d, r.x, r.y); codes4_scale(qb, bias, d, r.z, r.w); }
                }
                TC_OUT(4 * b + c, r);
            }
        }
    } else if constexpr (T == T_IQ4_XS) {
        // sub-blocks 2KS, 2KS+1 (32 values each, Q4_0 nibble order); words: d | scales_h, scales_l, qs from word 2
        const float dd = h2f(u[0] & 0xFFFF);
        const __half2 bias = __float2half2_rn(1152.0f);
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const int ib = 2 * KS + b;
            const __half2 d = __float2half2_rn(dd * (float)iq4xs_scale(u[0], u[1], ib));
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int hi = c >> 1;
                const uint32_t qa = u[2 + 4 * ib + 2 * (c & 1)] >> (4 * hi), qb = u[2 + 4 * ib + 2 * (c & 1) + 1] >> (4 * hi);
                uint4 r;
                codes4_scale(iq4nl_lookup4(qa) ^ 0x80808080u, bias, d, r.x, r.y); codes4_scale(iq4nl_lookup4(qb) ^ 0x80808080u, bias, d, r.z, r.w);
                TC_OUT(4 * b + c, r);
            }
        }
    } else if constexpr (T == T_Q2_K || T == T_Q3_K) {
        // K-step KS = half h = KS / 2, bit pairs jj0 = 2 (KS % 2) (chunks 0..3) and jj0 + 1 (chunks 4..7); chunk c: l = 8 (c % 4) ..
        constexpr bool THREE = (T == T_Q3_K);
        constexpr int h = KS >> 1, jj0 = 2 * (KS & 1);
        constexpr int QS0 = THREE ? 8 : 4;                       // first qs word (Q3_K: after hmask[32]; Q2_K: after scales[16])
        const float dd = THREE ? h2f(u[27] & 0xFFFF) : h2f(u[20] & 0xFFFF), dmn = THREE ? 0.0f : h2f(u[20] >> 16);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int jj = jj0 + (c >> 2), l0 = 8 * (c & 3), g16 = 8 * h + 2 * jj + (l0 >> 4);
            const uint32_t wa = u[QS0 + 8 * h + (l0 >> 2)], wb = u[QS0 + 8 * h + (l0 >> 2) + 1];
            uint32_t qa = (wa >> (2 * jj)) & 0x03030303u, qb = (wb >> (2 * jj)) & 0x03030303u;
            uint4 r;
            if constexpr (!THREE) {
                const int sc = (int)((u[g16 >> 2] >> (8 * (g16 & 3))) & 0xFF);
                const __half2 d = __float2half2_rn(dd * (float)(sc & 0x0F)), m = __float2half2_rn(-(dmn * (float)(sc >> 4)));
                codes4_affine(qa, d, m, r.x, r.y); codes4_affine(qb, d, m, r.z, r.w);
            } else {
                const int bit = 4 * h + jj;
                qa |= ((u[(l0 >> 2)] >> bit) & 0x01010101u) << 2;                    // high bit set: code + 4 (then - 4 for every code)
                qb |= ((u[(l0 >> 2) + 1] >> bit) & 0x01010101u) << 2;
                const int lo = g16 < 8 ? (int)((u[24 + (g16 >> 2)] >> (8 * (g16 & 3))) & 0x0F) : (int)((u[24 + ((g16 - 8) >> 2)] >> (8 * ((g16 - 8) & 3) + 4)) & 0x0F);
                const int hi2 = (int)((u[26] >> (8 * (g16 & 3) + 2 * (g16 >> 2))) & 3);
                const __half2 d = __float2half2_rn(dd * (float)((lo | (hi2 << 4)) - 32)), bias = __float2half2_rn(1028.0f);
                codes4_scale(qa, bias, d, r.x, r.y); codes4_scale(qb, bias, d, r.z, r.w);
            }
            TC_OUT(c, r);
        }
    } else {   // Q4_K / Q5_K: 64-chunk KS of the superblock: sub-blocks 2KS (low nibbles) and 2KS+1 (high nibbles)
        constexpr bool FIVE = (T == T_Q5_K);
        constexpr int qo = (FIVE ? 12 : 4) + 8 * KS;             // word offset of qs[32 KS]
        const uint32_t s0 = u[1], s1 = u[2], s2 = u[3];
        const float dd = h2f(u[0] & 0xFFFF), dm = h2f(u[0] >> 16);
#pragma unroll
        for (int hi = 0; hi < 2; ++hi) {
            int sc, mn;
            const int J = 2 * KS + hi;
            if (J < 4) { sc = (s0 >> (8 * J)) & 63; mn = (s1 >> (8 * J)) & 63; }
            else { const int jj = J - 4; sc = ((s2 >> (8 * jj)) & 0x0F) | (((s0 >> (8 * jj + 6)) & 3) << 4); mn = ((s2 >> (8 * jj + 4)) & 0x0F) | (((s1 >> (8 * jj + 6)) & 3) << 4); }
            const __half2 d = __float2half2_rn(dd * (float)sc), m = __float2half2_rn(-(dm * (float)mn));
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                uint32_t a = (u[qo + 2 * c] >> (4 * hi)) & 0x0F0F0F0F, b = (u[qo + 2 * c + 1] >> (4 * hi)) & 0x0F0F0F0F;
                if constexpr (FIVE) {
                    a |= ((u[4 + 2 * c] >> (2 * KS + hi)) & 0x01010101) << 4;       // qh words 4..11
                    b |= ((u[4 + 2 * c + 1] >> (2 * KS + hi)) & 0x01010101) << 4;
                }
                uint4 r;
                codes4_affine(a, d, m, r.x, r.y);
                codes4_affine(b, d, m, r.z, r.w);
                TC_OUT(4 * hi + c, r);
            }
        }
    }
}

} // namespace b200
