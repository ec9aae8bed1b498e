// b200_quants.cuh — packed block formats and the 64-element "unit" integer dot product (sm_90a).
//
// Weights stay in the reference's packed block_q* layout in HBM (consumed as-is, never repacked):
//   Q4_0 18 B / 32   (reference src/ggml-common.h:161-166)   Q8_0 34 B / 32   (:203-208)
//   Q4_K 144 B / 256 (:279-290)   Q5_K 176 B / 256 (:296-308)   Q6_K 210 B / 256 (:314-320)
// Activations are quantized on the fly to int8 exactly as the reference CPU backend does before its
// vec_dot (src/ggml-cpu/ggml-cpu.c:7490-7509): Q8_0-style (per 32, fp16-rounded scale; AVX2 flavour
// src/ggml-cpu/ggml-cpu-quants.c:778-835) for Q4_0/Q8_0 weights, Q8_K-style (per 256, f32 scale;
// src/ggml-quants.c:2479-2516) for the K-quants, so results match ggml-cpu up to f32 summation order.
//
// Work decomposition shared by every mat-vec kernel: a row is a sequence of UNITS of 64 weights.
//   Q4_0 / Q8_0 : unit u = blocks 2u, 2u+1               (36 B / 68 B, 4-byte aligned when K % 64 == 0)
//   Q4_K / Q5_K : unit u = superblock u/4, 64-chunk u%4  (32 B of qs [+ 32 B qh] + the 16 B header)
//   Q6_K        : unit u = superblock u/4, half (u/2)%2, l-range 16*(u%2): 4 groups of 16 weights
// A unit's activations are 4 pieces of 16 int8: contiguous for all formats but Q6_K (stride 32).
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace b200 {

// enum ggml_type ids (reference include/ggml.h:351-390)
enum : int { T_F32 = 0, T_F16 = 1, T_Q4_0 = 2, T_Q4_1 = 3, T_Q5_0 = 6, T_Q5_1 = 7, T_Q8_0 = 8, T_Q2_K = 10, T_Q3_K = 11, T_Q4_K = 12, T_Q5_K = 13, T_Q6_K = 14, T_IQ4_NL = 20, T_IQ4_XS = 23,
              T_IQ2_XXS = 16, T_IQ3_XXS = 18, T_IQ1_S = 19, T_IQ2_XS = 17, T_IQ3_S = 21, T_IQ2_S = 22, T_IQ1_M = 29, T_TQ1_0 = 34, T_TQ2_0 = 35 };

// The formats each kernel family is instantiated for.  A family's planning, workspace and launch code all dispatch through its one list.
template <int... Ts> struct format_list {};
// bandwidth mat-vec (mmvq_sb.cu, mmvq_mma.cu), tensor-core GEMM and grouped MUL_MAT_ID (mmq_tc2.cu)
using TC_FORMATS = format_list<T_Q4_0, T_Q8_0, T_Q4_K, T_Q5_K, T_Q6_K, T_Q4_1, T_Q5_0, T_Q5_1, T_IQ4_NL, T_IQ4_XS, T_Q2_K, T_Q3_K>;
// first-generation TMA mat-vec (mmvq_tma_kernel)
using TMA_FORMATS = format_list<T_Q4_0, T_Q8_0, T_Q4_K, T_Q5_K, T_Q6_K>;
// every block format: generic mat-vec, mmid_kernel, dequantize_kernel
using ALL_FORMATS = format_list<T_Q4_0, T_Q8_0, T_Q4_K, T_Q5_K, T_Q6_K, T_Q4_1, T_Q5_0, T_Q5_1, T_Q2_K, T_Q3_K, T_IQ4_NL, T_IQ4_XS,
                                T_IQ2_XXS, T_IQ3_XXS, T_IQ1_S, T_IQ2_XS, T_IQ2_S, T_IQ3_S, T_IQ1_M, T_TQ1_0, T_TQ2_0>;

// Calls f(std::integral_constant<int, T>()) for the format T of the list that equals `type`; false when the list does not hold it.
template <int... Ts, typename F> inline bool with_format(format_list<Ts...>, int type, F && f) {
    return ((type == Ts ? (f(std::integral_constant<int, Ts>()), true) : false) || ...);
}

template <int T> struct fmt;
template <> struct fmt<T_Q4_0> { static constexpr int QK = 32,  BYTES = 18,  ACT_K = 0; };
template <> struct fmt<T_Q8_0> { static constexpr int QK = 32,  BYTES = 34,  ACT_K = 0; };
template <> struct fmt<T_Q4_K> { static constexpr int QK = 256, BYTES = 144, ACT_K = 1; };
template <> struct fmt<T_Q5_K> { static constexpr int QK = 256, BYTES = 176, ACT_K = 1; };
template <> struct fmt<T_Q6_K> { static constexpr int QK = 256, BYTES = 210, ACT_K = 1; };
// SURVEY §8f-2 formats (generic mat-vec / MUL_MAT_ID / dequantize paths; decode logic checked on the host by tests/hostemu):
//   Q4_1 20 B / 32 (src/ggml-common.h:168-180)   Q5_0 22 B / 32 (:182-188)   Q5_1 24 B / 32 (:190-203)
//   Q2_K 84 B / 256 (:247-262)   Q3_K 110 B / 256 (:264-276)
// Q4_1 / Q5_1 carry a per-block minimum: the CPU backend pairs them with Q8_1 activations (d and s = d * sum of codes).
template <> struct fmt<T_Q4_1> { static constexpr int QK = 32,  BYTES = 20,  ACT_K = 0; };
template <> struct fmt<T_Q5_0> { static constexpr int QK = 32,  BYTES = 22,  ACT_K = 0; };
template <> struct fmt<T_Q5_1> { static constexpr int QK = 32,  BYTES = 24,  ACT_K = 0; };
template <> struct fmt<T_Q2_K> { static constexpr int QK = 256, BYTES = 84,  ACT_K = 1; };
template <> struct fmt<T_Q3_K> { static constexpr int QK = 256, BYTES = 110, ACT_K = 1; };
// IQ4_NL (src/ggml-common.h:398-403): the Q4_0 layout, the nibble indexes a fixed non-linear int8 codebook (kvalues_iq4nl, src/ggml-quants.c:2434)
template <> struct fmt<T_IQ4_NL> { static constexpr int QK = 32, BYTES = 18, ACT_K = 0; };
// IQ4_XS (:406-411): 136 B / 256 = d, scales_h (u16), scales_l[4], qs[128]; eight 32-value sub-blocks with 6-bit scales (value - 32), same codebook
template <> struct fmt<T_IQ4_XS> { static constexpr int QK = 256, BYTES = 136, ACT_K = 1; };
// grid-codebook i-quants (b200_iq.cuh): generic mat-vec / MUL_MAT_ID / dequantize kernels
template <> struct fmt<T_IQ2_XXS> { static constexpr int QK = 256, BYTES = 66, ACT_K = 1; };
template <> struct fmt<T_IQ3_XXS> { static constexpr int QK = 256, BYTES = 98, ACT_K = 1; };
template <> struct fmt<T_IQ1_S>   { static constexpr int QK = 256, BYTES = 50, ACT_K = 1; };
template <> struct fmt<T_IQ2_XS>  { static constexpr int QK = 256, BYTES = 74, ACT_K = 1; };
template <> struct fmt<T_IQ2_S>   { static constexpr int QK = 256, BYTES = 82, ACT_K = 1; };
template <> struct fmt<T_IQ3_S>   { static constexpr int QK = 256, BYTES = 110, ACT_K = 1; };
template <> struct fmt<T_IQ1_M>   { static constexpr int QK = 256, BYTES = 56, ACT_K = 1; };
template <> struct fmt<T_TQ1_0>   { static constexpr int QK = 256, BYTES = 54, ACT_K = 1; };
template <> struct fmt<T_TQ2_0>   { static constexpr int QK = 256, BYTES = 66, ACT_K = 1; };

__host__ __device__ inline int    type_qk(int t)    { return t == T_Q4_0 || t == T_Q8_0 || t == T_Q4_1 || t == T_Q5_0 || t == T_Q5_1 || t == T_IQ4_NL ? 32 : 256; }
__host__ __device__ inline int    type_bytes(int t) {
    return t == T_Q4_0 ? 18 : t == T_Q8_0 ? 34 : t == T_Q4_K ? 144 : t == T_Q5_K ? 176 : t == T_Q6_K ? 210
         : t == T_Q4_1 ? 20 : t == T_Q5_0 ? 22 : t == T_Q5_1 ? 24 : t == T_Q2_K ? 84 : t == T_Q3_K ? 110 : t == T_IQ4_NL ? 18 : t == T_IQ4_XS ? 136
         : t == T_IQ2_XXS ? 66 : t == T_IQ3_XXS ? 98 : t == T_IQ1_S ? 50
         : t == T_IQ2_XS ? 74 : t == T_IQ2_S ? 82 : t == T_IQ3_S ? 110 : t == T_IQ1_M ? 56 : t == T_TQ1_0 ? 54 : t == T_TQ2_0 ? 66 : 0;
}
__host__ __device__ inline bool   type_is_kquant(int t) { return t == T_Q4_K || t == T_Q5_K || t == T_Q6_K || t == T_Q2_K || t == T_Q3_K || t == T_IQ4_XS || t == T_IQ2_XXS || t == T_IQ3_XXS || t == T_IQ1_S
                                                               || t == T_IQ2_XS || t == T_IQ2_S || t == T_IQ3_S || t == T_IQ1_M || t == T_TQ1_0 || t == T_TQ2_0; }   // Q8_K activations
__host__ __device__ inline size_t row_bytes(int t, int64_t k) { return (size_t)(k / type_qk(t)) * type_bytes(t); }

// ------------------------------------------------------------------ quantized activation record
// One record per activation row (K values), the same for both families:
//   q   : int8[K]
//   bs  : int16[K/16]   sums of q over groups of 16 (block_q8_K.bsums; also gives Q4_0's "-8" term)
//   d   : float[K/32] (fp16-rounded, Q8_0 family) or float[K/256] (Q8_K family)
//   s   : float[K/32], Q8_0 family only: block_q8_1.s = fp16(d_unrounded * sum of the block's codes), for weights with a minimum
// laid out q | bs | d | s, each part 16-byte aligned.
#define B200_ACT_HAS_S 1
struct act_layout {
    int32_t off_bs, off_d, off_s, bytes;
};
__host__ __device__ inline act_layout make_act_layout(int64_t K, bool kq) {
    act_layout L;
    L.off_bs = (int32_t)((K + 15) & ~(int64_t)15);
    L.off_d  = L.off_bs + (int32_t)(((K / 16) * 2 + 15) & ~(int64_t)15);
    L.off_s  = L.off_d + (int32_t)((((kq ? K / 256 : K / 32)) * 4 + 15) & ~(int64_t)15);
    L.bytes  = L.off_s + (kq ? 0 : (int32_t)(((K / 32) * 4 + 15) & ~(int64_t)15));
    return L;
}

// ------------------------------------------------------------------ small helpers
// GELU exactly as the CPU backend evaluates it: through an fp16 -> fp16 table (ggml_vec_gelu_f32, src/ggml-cpu/ggml-cpu.c:1355 ff.)
__device__ __forceinline__ float gelu_ggml(float v) {
    if (v <= -10.0f) return 0.0f;
    if (v >= 10.0f) return v;
    const float xh = __half2float(__float2half_rn(v));
    const float g = 0.5f * xh * (1.0f + tanhf(0.79788456080286535587989211986876f * xh * (1.0f + 0.044715f * xh * xh)));
    return __half2float(__float2half_rn(g));
}
// GELU_QUICK likewise through ggml-cpu's fp16 -> fp16 table of x * (1 / (1 + expf(-1.702 x))) (ggml_vec_gelu_quick_f32, ggml-cpu.c:1797).
// It has no cut-offs: |x| >= 65520 reads the table at +-inf, which gives +inf above and NaN (-inf * 0) below.
__device__ __forceinline__ float gelu_quick_ggml(float v) {
    const float xh = __half2float(__float2half_rn(v));
    return __half2float(__float2half_rn(xh * (1.0f / (1.0f + expf(-1.702f * xh)))));
}
__device__ __forceinline__ float h2f(uint32_t bits16) { return __half2float(__ushort_as_half((unsigned short)bits16)); }

// n consecutive 32-bit words starting at a 2-byte aligned address (generic/global/shared)
template <int N> __device__ __forceinline__ void load_words_a2(const uint8_t * p, uint32_t (&w)[N]) {
    const uintptr_t a = (uintptr_t)p;
    const uint32_t * q = (const uint32_t *)(a & ~(uintptr_t)3);
    if (a & 2) {
        uint32_t prev = q[0];
#pragma unroll
        for (int i = 0; i < N; ++i) { const uint32_t nxt = q[i + 1]; w[i] = __funnelshift_r(prev, nxt, 16); prev = nxt; }
    } else {
#pragma unroll
        for (int i = 0; i < N; ++i) w[i] = q[i];
    }
}
__device__ __forceinline__ uint32_t load_u16(const uint8_t * p) { return *(const uint16_t *)p; }

// activations of one unit, shared by every weight row processed against it
struct unit_act {
    int   q[16];   // 64 int8
    int   bs[4];   // sums of the four groups of 16
    float d[2];    // Q8_0 family: scales of the two 32-blocks; Q8_K family: d[0] = superblock scale
    float s[2];    // Q8_1's s of the two 32-blocks (only loaded for weight formats with a minimum)
};
template <int T> struct needs_s { static constexpr bool value = (T == T_Q4_1 || T == T_Q5_1); };

// k offset of 16-piece g of unit u
template <int T> __device__ __forceinline__ int unit_piece_k(int u, int g) {
    if constexpr (T == T_Q6_K) return (u >> 2) * 256 + ((u >> 1) & 1) * 128 + (u & 1) * 16 + g * 32;
    else                       return u * 64 + g * 16;
}

template <int T> __device__ __forceinline__ void load_unit_act(const uint8_t * rec, const act_layout & L, int u, unit_act & A) {
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        const int k = unit_piece_k<T>(u, g);
        const int4 v = *(const int4 *)(rec + k);
        A.q[4 * g + 0] = v.x; A.q[4 * g + 1] = v.y; A.q[4 * g + 2] = v.z; A.q[4 * g + 3] = v.w;
        A.bs[g] = *(const int16_t *)(rec + L.off_bs + (k >> 4) * 2);
    }
    const float * d = (const float *)(rec + L.off_d);
    if constexpr (fmt<T>::ACT_K) { A.d[0] = d[u >> 2]; A.d[1] = 0.0f; }
    else                        { A.d[0] = d[2 * u]; A.d[1] = d[2 * u + 1]; }
    if constexpr (needs_s<T>::value) { const float * sv = (const float *)(rec + L.off_s); A.s[0] = sv[2 * u]; A.s[1] = sv[2 * u + 1]; }
    else                             { A.s[0] = 0.0f; A.s[1] = 0.0f; }
}

// ------------------------------------------------------------------ unit dot products
// `row` points at the first byte of a weight row (2-byte aligned; 16-byte aligned for Q4_K/Q5_K).
// Returns this unit's contribution to dot(row, activation) in f32.

__device__ __forceinline__ int dp4a_s(int a, int b, int c) { return __dp4a(a, b, c); }

// Q4_K / Q5_K: 6-bit (scale, min) pair j of the 12-byte packing (reference get_scale_min_k4, ggml-quants.c:631-638)
__device__ __forceinline__ void k4_scale_min(const uint32_t (&s)[3], int j, int & sc, int & mn) {
    // s[0] = bytes 0..3, s[1] = bytes 4..7, s[2] = bytes 8..11
    if (j < 4) {
        sc = (s[0] >> (8 * j)) & 63;
        mn = (s[1] >> (8 * j)) & 63;
    } else {
        const int jj = j - 4;
        const uint32_t b8 = (s[2] >> (8 * jj)) & 0xFF;
        sc = (b8 & 0x0F) | (((s[0] >> (8 * jj + 6)) & 3) << 4);
        mn = (b8 >> 4)   | (((s[1] >> (8 * jj + 6)) & 3) << 4);
    }
}

template <int T> __device__ __forceinline__ float unit_dot(const uint8_t * row, int u, const unit_act & A);

template <> __device__ __forceinline__ float unit_dot<T_Q4_0>(const uint8_t * row, int u, const unit_act & A) {
    uint32_t w[9];
    load_words_a2<9>(row + 36 * u, w);
    // block 0: d = w0[15:0], qs = bytes 2..17 ; block 1: d = w4[31:16], qs = w5..w8
    uint32_t qa[4], qb[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { qa[i] = __funnelshift_r(w[i], w[i + 1], 16); qb[i] = w[5 + i]; }
    int s0 = 0, s1 = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        s0 = dp4a_s(qa[i] & 0x0F0F0F0F,        A.q[i],      s0);
        s0 = dp4a_s((qa[i] >> 4) & 0x0F0F0F0F, A.q[4 + i],  s0);
        s1 = dp4a_s(qb[i] & 0x0F0F0F0F,        A.q[8 + i],  s1);
        s1 = dp4a_s((qb[i] >> 4) & 0x0F0F0F0F, A.q[12 + i], s1);
    }
    s0 -= 8 * (A.bs[0] + A.bs[1]);
    s1 -= 8 * (A.bs[2] + A.bs[3]);
    const float d0 = h2f(w[0] & 0xFFFF), d1 = h2f(w[4] >> 16);
    return (float)s0 * d0 * A.d[0] + (float)s1 * d1 * A.d[1];
}

template <> __device__ __forceinline__ float unit_dot<T_Q8_0>(const uint8_t * row, int u, const unit_act & A) {
    uint32_t w[17];
    load_words_a2<17>(row + 68 * u, w);
    int s0 = 0, s1 = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        s0 = dp4a_s((int)__funnelshift_r(w[i], w[i + 1], 16), A.q[i], s0);
        s1 = dp4a_s((int)w[9 + i], A.q[8 + i], s1);
    }
    const float d0 = h2f(w[0] & 0xFFFF), d1 = h2f(w[8] >> 16);
    return (float)s0 * (d0 * A.d[0]) + (float)s1 * (d1 * A.d[1]);
}

template <> __device__ __forceinline__ float unit_dot<T_Q4_K>(const uint8_t * row, int u, const unit_act & A) {
    const uint8_t * sb = row + 144 * (u >> 2);
    const int c = u & 3;
    const uint4 hdr = *(const uint4 *)sb;                   // d | dmin | scales[12]
    const uint4 qa = *(const uint4 *)(sb + 16 + 32 * c), qb = *(const uint4 *)(sb + 32 + 32 * c);
    const uint32_t q[8] = { qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w };
    int p0 = 0, p1 = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        p0 = dp4a_s(q[i] & 0x0F0F0F0F,        A.q[i],     p0);
        p1 = dp4a_s((q[i] >> 4) & 0x0F0F0F0F, A.q[8 + i], p1);
    }
    const uint32_t s[3] = { hdr.y, hdr.z, hdr.w };
    int sc0, m0, sc1, m1;
    k4_scale_min(s, 2 * c, sc0, m0);
    k4_scale_min(s, 2 * c + 1, sc1, m1);
    const float d = h2f(hdr.x & 0xFFFF) * A.d[0], dmin = h2f(hdr.x >> 16) * A.d[0];
    return d * (float)(sc0 * p0 + sc1 * p1) - dmin * (float)(m0 * (A.bs[0] + A.bs[1]) + m1 * (A.bs[2] + A.bs[3]));
}

template <> __device__ __forceinline__ float unit_dot<T_Q5_K>(const uint8_t * row, int u, const unit_act & A) {
    const uint8_t * sb = row + 176 * (u >> 2);
    const int c = u & 3;
    const uint4 hdr = *(const uint4 *)sb;                   // d | dmin | scales[12]
    const uint4 ha = *(const uint4 *)(sb + 16), hb = *(const uint4 *)(sb + 32);      // qh[32]
    const uint4 qa = *(const uint4 *)(sb + 48 + 32 * c), qb = *(const uint4 *)(sb + 64 + 32 * c);
    const uint32_t q[8] = { qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w };
    const uint32_t h[8] = { ha.x, ha.y, ha.z, ha.w, hb.x, hb.y, hb.z, hb.w };
    int p0 = 0, p1 = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint32_t hi = h[i] >> (2 * c);
        p0 = dp4a_s((q[i] & 0x0F0F0F0F)        | ((hi & 0x01010101) << 4), A.q[i],     p0);
        p1 = dp4a_s(((q[i] >> 4) & 0x0F0F0F0F) | ((hi & 0x02020202) << 3), A.q[8 + i], p1);
    }
    const uint32_t s[3] = { hdr.y, hdr.z, hdr.w };
    int sc0, m0, sc1, m1;
    k4_scale_min(s, 2 * c, sc0, m0);
    k4_scale_min(s, 2 * c + 1, sc1, m1);
    const float d = h2f(hdr.x & 0xFFFF) * A.d[0], dmin = h2f(hdr.x >> 16) * A.d[0];
    return d * (float)(sc0 * p0 + sc1 * p1) - dmin * (float)(m0 * (A.bs[0] + A.bs[1]) + m1 * (A.bs[2] + A.bs[3]));
}

template <> __device__ __forceinline__ float unit_dot<T_Q6_K>(const uint8_t * row, int u, const unit_act & A) {
    const uint8_t * sb = row + 210 * (u >> 2);
    const int h = (u >> 1) & 1, j = u & 1;
    uint32_t la[4], lb[4], qh[4], sw[2];
    load_words_a2<4>(sb + 64 * h + 16 * j, la);             // ql[64h + l],      l = 16j .. 16j+15
    load_words_a2<4>(sb + 64 * h + 32 + 16 * j, lb);        // ql[64h + 32 + l]
    load_words_a2<4>(sb + 128 + 32 * h + 16 * j, qh);       // qh[32h + l]
    load_words_a2<2>(sb + 192 + 8 * h, sw);                 // scales[8h .. 8h+7]
    int p[4] = { 0, 0, 0, 0 };
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        p[0] = dp4a_s((la[i] & 0x0F0F0F0F)        | ((qh[i] << 4) & 0x30303030), A.q[i],      p[0]);
        p[1] = dp4a_s((lb[i] & 0x0F0F0F0F)        | ((qh[i] << 2) & 0x30303030), A.q[4 + i],  p[1]);
        p[2] = dp4a_s(((la[i] >> 4) & 0x0F0F0F0F) | ( qh[i]       & 0x30303030), A.q[8 + i],  p[2]);
        p[3] = dp4a_s(((lb[i] >> 4) & 0x0F0F0F0F) | ((qh[i] >> 2) & 0x30303030), A.q[12 + i], p[3]);
    }
    int tot = 0;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        const int idx = j + 2 * g;                                            // scales[8h + j + 2g]
        const int sc = (int)(int8_t)((sw[idx >> 2] >> (8 * (idx & 3))) & 0xFF);
        tot += sc * (p[g] - 32 * A.bs[g]);
    }
    const float d = h2f(load_u16(sb + 208)) * A.d[0];
    return d * (float)tot;
}

// ---- SURVEY §8f-2 formats ------------------------------------------------------------------------------------------------
// four fifth-bits (bits 0..3 of x) -> bit 4 of the four bytes of a word
__device__ __forceinline__ uint32_t spread4_to_bit4(uint32_t x) { return (((x & 0xF) * 0x00204081u) & 0x01010101u) << 4; }

// dot of the 32 5-bit codes of a Q5 block (nibble words q[4], fifth bits qh) with the block's 32 int8 activations
__device__ __forceinline__ int q5_block_dot(const uint32_t (&q)[4], uint32_t qh, const int * y) {
    int s = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        s = dp4a_s((int)((q[i] & 0x0F0F0F0F)        | spread4_to_bit4(qh >> (4 * i))),      y[i],     s);   // elements 4i .. 4i+3
        s = dp4a_s((int)(((q[i] >> 4) & 0x0F0F0F0F) | spread4_to_bit4(qh >> (16 + 4 * i))), y[4 + i], s);   // elements 16+4i ..
    }
    return s;
}

template <> __device__ __forceinline__ float unit_dot<T_Q4_1>(const uint8_t * row, int u, const unit_act & A) {
    uint32_t w[10];
    load_words_a2<10>(row + 40 * u, w);                    // block: d | m, qs[16]
    int s0 = 0, s1 = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        s0 = dp4a_s(w[1 + i] & 0x0F0F0F0F,        A.q[i],      s0);
        s0 = dp4a_s((w[1 + i] >> 4) & 0x0F0F0F0F, A.q[4 + i],  s0);
        s1 = dp4a_s(w[6 + i] & 0x0F0F0F0F,        A.q[8 + i],  s1);
        s1 = dp4a_s((w[6 + i] >> 4) & 0x0F0F0F0F, A.q[12 + i], s1);
    }
    return (h2f(w[0] & 0xFFFF) * A.d[0]) * (float)s0 + h2f(w[0] >> 16) * A.s[0]
         + (h2f(w[5] & 0xFFFF) * A.d[1]) * (float)s1 + h2f(w[5] >> 16) * A.s[1];
}

template <> __device__ __forceinline__ float unit_dot<T_Q5_0>(const uint8_t * row, int u, const unit_act & A) {
    uint32_t w[11];
    load_words_a2<11>(row + 44 * u, w);                    // block: d (2 B), qh (4 B), qs[16]; the second block starts at byte 22
    uint32_t qa[4], qb[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { qa[i] = __funnelshift_r(w[1 + i], w[2 + i], 16); qb[i] = w[7 + i]; }
    const uint32_t qha = __funnelshift_r(w[0], w[1], 16), qhb = w[6];
    const int s0 = q5_block_dot(qa, qha, A.q)     - 16 * (A.bs[0] + A.bs[1]);
    const int s1 = q5_block_dot(qb, qhb, A.q + 8) - 16 * (A.bs[2] + A.bs[3]);
    return (h2f(w[0] & 0xFFFF) * A.d[0]) * (float)s0 + (h2f(w[5] >> 16) * A.d[1]) * (float)s1;
}

template <> __device__ __forceinline__ float unit_dot<T_Q5_1>(const uint8_t * row, int u, const unit_act & A) {
    uint32_t w[12];
    load_words_a2<12>(row + 48 * u, w);                    // block: d | m, qh, qs[16]
    const uint32_t qa[4] = { w[2], w[3], w[4], w[5] }, qb[4] = { w[8], w[9], w[10], w[11] };
    const int s0 = q5_block_dot(qa, w[1], A.q), s1 = q5_block_dot(qb, w[7], A.q + 8);
    return (h2f(w[0] & 0xFFFF) * A.d[0]) * (float)s0 + h2f(w[0] >> 16) * A.s[0]
         + (h2f(w[6] & 0xFFFF) * A.d[1]) * (float)s1 + h2f(w[6] >> 16) * A.s[1];
}

// IQ4_NL codebook, four int8 entries per word (little endian): { -127, -104, -83, -65, -49, -35, -22, -10, 1, 13, 25, 38, 53, 69, 89, 113 }
#define B200_IQ4NL_W0 0xBFAD9881u
#define B200_IQ4NL_W1 0xF6EADDCFu
#define B200_IQ4NL_W2 0x26190D01u
#define B200_IQ4NL_W3 0x71594535u
__device__ __forceinline__ int iq4nl_value(int n) {              // codebook[n], n = 0..15
    const uint32_t w = n < 4 ? B200_IQ4NL_W0 : n < 8 ? B200_IQ4NL_W1 : n < 12 ? B200_IQ4NL_W2 : B200_IQ4NL_W3;
    return (int)(int8_t)((w >> (8 * (n & 3))) & 0xFF);
}
// four nibbles (low nibble of each byte of x) -> their four int8 codebook entries, one per byte: two 8-entry byte permutes
// (selector = nibble & 7) and a per-byte choice by bit 3 of the nibble
__device__ __forceinline__ uint32_t iq4nl_lookup4(uint32_t x) {
    const uint32_t q7 = x & 0x07070707u;
    const uint32_t sel = (q7 & 0x7u) | ((q7 >> 4) & 0x70u) | ((q7 >> 8) & 0x700u) | ((q7 >> 12) & 0x7000u);
    const uint32_t lo = __byte_perm(B200_IQ4NL_W0, B200_IQ4NL_W1, sel), hi = __byte_perm(B200_IQ4NL_W2, B200_IQ4NL_W3, sel);
    const uint32_t m = ((x >> 3) & 0x01010101u) * 0xFFu;        // 0xFF in the bytes whose nibble is >= 8
    return (lo & ~m) | (hi & m);
}
template <> __device__ __forceinline__ float unit_dot<T_IQ4_NL>(const uint8_t * row, int u, const unit_act & A) {
    uint32_t w[9];
    load_words_a2<9>(row + 36 * u, w);                     // as Q4_0: block 0 d = w0[15:0], qs bytes 2..17; block 1 d = w4[31:16], qs = w5..w8
    int s0 = 0, s1 = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const uint32_t qa = __funnelshift_r(w[i], w[i + 1], 16), qb = w[5 + i];
        s0 = dp4a_s((int)iq4nl_lookup4(qa),      A.q[i],      s0);
        s0 = dp4a_s((int)iq4nl_lookup4(qa >> 4), A.q[4 + i],  s0);
        s1 = dp4a_s((int)iq4nl_lookup4(qb),      A.q[8 + i],  s1);
        s1 = dp4a_s((int)iq4nl_lookup4(qb >> 4), A.q[12 + i], s1);
    }
    return (A.d[0] * h2f(w[0] & 0xFFFF)) * (float)s0 + (A.d[1] * h2f(w[4] >> 16)) * (float)s1;
}

// 6-bit scale (biased by 32) of sub-block ib of an IQ4_XS superblock: w0 = d | scales_h << 16, w1 = scales_l[4]
__device__ __forceinline__ int iq4xs_scale(uint32_t w0, uint32_t w1, int ib) {
    return (int)(((w1 >> (4 * ib)) & 0x0F) | ((((w0 >> 16) >> (2 * ib)) & 3) << 4)) - 32;
}
template <> __device__ __forceinline__ float unit_dot<T_IQ4_XS>(const uint8_t * row, int u, const unit_act & A) {
    const uint8_t * sb = row + 136 * (u >> 2);              // 8-byte aligned superblocks
    const int c = u & 3;                                    // sub-blocks 2c, 2c+1: 32 bytes of qs at 8 + 32 c
    uint32_t hd[2], q[8];
    load_words_a2<2>(sb, hd);
    load_words_a2<8>(sb + 8 + 32 * c, q);
    int tot = 0;
#pragma unroll
    for (int k = 0; k < 2; ++k) {                           // sub-block 2c + k: low nibbles = its elements 0..15 (piece 2k), high = 16..31 (piece 2k+1)
        int s = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            s = dp4a_s((int)iq4nl_lookup4(q[4 * k + i]),      A.q[8 * k + i],     s);
            s = dp4a_s((int)iq4nl_lookup4(q[4 * k + i] >> 4), A.q[8 * k + 4 + i], s);
        }
        tot += iq4xs_scale(hd[0], hd[1], 2 * c + k) * s;
    }
    return (h2f(hd[0] & 0xFFFF) * A.d[0]) * (float)tot;
}

// byte k of a little-endian word array
template <int N> __device__ __forceinline__ int word_byte(const uint32_t (&w)[N], int k) { return (int)((w[k >> 2] >> (8 * (k & 3))) & 0xFF); }

// Q2_K / Q3_K: element 128 h + 32 j + l of a superblock has its 2-bit code in bits 2j..2j+1 of qs[32 h + l] and belongs to the
// 16-element group 8 h + 2 j + l / 16.  Unit u (64 weights) = half h = (u % 4) / 2, bit pairs j0 = 2 (u % 2) and j0 + 1;
// its pieces g = 0..3 are (j0, l < 16), (j0, l >= 16), (j0 + 1, l < 16), (j0 + 1, l >= 16): contiguous activations.
template <> __device__ __forceinline__ float unit_dot<T_Q2_K>(const uint8_t * row, int u, const unit_act & A) {
    const uint8_t * sb = row + 84 * (u >> 2);               // scales[16] @0, qs[64] @16, d @80, dmin @82
    const int h = (u >> 1) & 1, j0 = 2 * (u & 1);
    uint32_t sc[4], q[8];
    load_words_a2<4>(sb, sc);
    load_words_a2<8>(sb + 16 + 32 * h, q);
    int isum = 0, msum = 0;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        const int jj = j0 + (g >> 1), half16 = g & 1;
        int p = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) p = dp4a_s((int)((q[4 * half16 + i] >> (2 * jj)) & 0x03030303), A.q[4 * g + i], p);
        const int s = word_byte(sc, 8 * h + 2 * jj + half16);
        isum += (s & 0x0F) * p;
        msum += (s >> 4) * A.bs[g];
    }
    const float dall = A.d[0] * h2f(load_u16(sb + 80)), dmin = A.d[0] * h2f(load_u16(sb + 82));
    return dall * (float)isum - dmin * (float)msum;
}

template <> __device__ __forceinline__ float unit_dot<T_Q3_K>(const uint8_t * row, int u, const unit_act & A) {
    const uint8_t * sb = row + 110 * (u >> 2);              // hmask[32] @0, qs[64] @32, scales[12] @96, d @108 (2-byte aligned)
    const int h = (u >> 1) & 1, j0 = 2 * (u & 1);
    uint32_t hm[8], q[8], sc[3];
    load_words_a2<8>(sb, hm);
    load_words_a2<8>(sb + 32 + 32 * h, q);
    load_words_a2<3>(sb + 96, sc);
    int isum = 0;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        const int jj = j0 + (g >> 1), half16 = g & 1, bit = 4 * h + jj;
        int p = 0, low = 0;                                  // low = sum of the activations whose high bit is clear (code - 4)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            p   = dp4a_s((int)((q[4 * half16 + i] >> (2 * jj)) & 0x03030303), A.q[4 * g + i], p);
            low = dp4a_s((int)(~(hm[4 * half16 + i] >> bit) & 0x01010101),    A.q[4 * g + i], low);
        }
        const int g16 = 8 * h + 2 * jj + half16;
        const int lo = g16 < 8 ? (word_byte(sc, g16) & 0x0F) : (word_byte(sc, g16 - 8) >> 4);
        const int hi = (word_byte(sc, 8 + (g16 & 3)) >> (2 * (g16 >> 2))) & 3;
        isum += ((lo | (hi << 4)) - 32) * (p - 4 * low);
    }
    return (h2f(load_u16(sb + 108)) * A.d[0]) * (float)isum;
}

// single trailing 32-block of a row of a 32-element-block format whose block count is odd (K % 64 == 32)
template <int T> __device__ __forceinline__ float tail_block_dot(const uint8_t * blk, const uint8_t * rec, const act_layout & L, int kblk) {
    const int * aq = (const int *)(rec + kblk * 32);
    const float ad = ((const float *)(rec + L.off_d))[kblk];
    int s = 0;
    if constexpr (T == T_Q4_0) {
        uint32_t w[5];
        load_words_a2<5>(blk, w);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t q = __funnelshift_r(w[i], w[i + 1], 16);
            s = __dp4a((int)(q & 0x0F0F0F0F), aq[i], s);
            s = __dp4a((int)((q >> 4) & 0x0F0F0F0F), aq[4 + i], s);
        }
        const int16_t * bs = (const int16_t *)(rec + L.off_bs);
        s -= 8 * (bs[2 * kblk] + bs[2 * kblk + 1]);
        return (float)s * h2f(w[0] & 0xFFFF) * ad;
    } else if constexpr (T == T_Q8_0) {
        uint32_t w[9];
        load_words_a2<9>(blk, w);
#pragma unroll
        for (int i = 0; i < 8; ++i) s = __dp4a((int)__funnelshift_r(w[i], w[i + 1], 16), aq[i], s);
        return (float)s * (h2f(w[0] & 0xFFFF) * ad);
    } else {
        // the other 32-block formats: the unit dot product on a private copy of the block followed by an all-zero block
        // (zero scale and minimum: contributes exactly 0) against a unit whose second half is zero
        __align__(4) uint8_t tmp[2 * fmt<T>::BYTES + 8];
#pragma unroll
        for (int i = 0; i < 2 * fmt<T>::BYTES + 8; ++i) tmp[i] = i < fmt<T>::BYTES ? blk[i] : (uint8_t)0;
        unit_act A;
        const int16_t * bs = (const int16_t *)(rec + L.off_bs);
#pragma unroll
        for (int i = 0; i < 8; ++i) { A.q[i] = aq[i]; A.q[8 + i] = 0; }
        A.bs[0] = bs[2 * kblk]; A.bs[1] = bs[2 * kblk + 1]; A.bs[2] = 0; A.bs[3] = 0;
        A.d[0] = ad; A.d[1] = 0.0f;
        A.s[0] = needs_s<T>::value ? ((const float *)(rec + L.off_s))[kblk] : 0.0f; A.s[1] = 0.0f;
        return unit_dot<T>(tmp, 0, A);
    }
}

// ------------------------------------------------------------------ activation quantizers (device)
__device__ __forceinline__ float4 load_f4(const float * p) {
    if (((uintptr_t)p & 15) == 0) return *(const float4 *)p;
    return make_float4(p[0], p[1], p[2], p[3]);
}

// One warp quantizes 256 consecutive activations x[0..255] (a Q8_K superblock, or eight Q8_0 blocks):
// lane l holds x[4l..4l+3] and x[128+4l..128+4l+3].  `kvalid` = number of valid elements (multiple of 32).

// Q8_0 family, AVX2 flavour: d = fp16(amax/127), q = rne(x * (127/amax))
__device__ __forceinline__ void warp_quantize_q8_0_x256(const float * x, int kvalid, uint8_t * rec, const act_layout & L, int k0) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int k = half * 128 + 4 * lane;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < kvalid) v = load_f4(x + k);
        float amax = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        const float id = amax != 0.0f ? __fdiv_rn(127.0f, amax) : 0.0f;
        const int q0 = __float2int_rn(v.x * id), q1 = __float2int_rn(v.y * id), q2 = __float2int_rn(v.z * id), q3 = __float2int_rn(v.w * id);
        int s = q0 + q1 + q2 + q3;
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);      // sum over 16 elements (4 lanes)
        const int s32 = s + __shfl_xor_sync(0xffffffffu, s, 4);                      // sum over the 32-block (8 lanes); all lanes take part
        if (k < kvalid) {
            *(uint32_t *)(rec + k0 + k) = (uint32_t)(q0 & 0xFF) | ((uint32_t)(q1 & 0xFF) << 8) | ((uint32_t)(q2 & 0xFF) << 16) | ((uint32_t)(q3 & 0xFF) << 24);
            if ((lane & 3) == 0) *(int16_t *)(rec + L.off_bs + ((k0 + k) >> 4) * 2) = (int16_t)s;
            if ((lane & 7) == 0) {
                const float dun = __fdiv_rn(amax, 127.0f);                                // block_q8_1: d = fp16(dun), s = fp16(dun * sum)
                ((float *)(rec + L.off_d))[(k0 + k) >> 5] = __half2float(__float2half_rn(dun));
                ((float *)(rec + L.off_s))[(k0 + k) >> 5] = __half2float(__float2half_rn(__fmul_rn(dun, (float)s32)));
            }
        }
    }
}

// Q8_K family: iscale = -127/max (max = the first element of largest magnitude), q = min(127, rne(iscale*x)), d = 1/iscale
__device__ __forceinline__ void warp_quantize_q8_K_x256(const float * x, uint8_t * rec, const act_layout & L, int k0) {
    const int lane = threadIdx.x & 31;
    const float4 a = load_f4(x + 4 * lane), b = load_f4(x + 128 + 4 * lane);
    const float v[8] = { a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w };
    float amax = 0.0f, vmax = 0.0f; int imax = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int idx = (i < 4 ? 4 * lane + i : 128 + 4 * lane + (i - 4));
        const float ax = fabsf(v[i]);
        if (ax > amax || (ax == amax && ax != 0.0f && idx < imax)) { amax = ax; vmax = v[i]; imax = idx; }
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float oa = __shfl_xor_sync(0xffffffffu, amax, o), ov = __shfl_xor_sync(0xffffffffu, vmax, o);
        const int   oi = __shfl_xor_sync(0xffffffffu, imax, o);
        if (oa > amax || (oa == amax && oi < imax)) { amax = oa; vmax = ov; imax = oi; }
    }
    int q[8];
    float d = 0.0f;
    if (amax != 0.0f) {
        const float iscale = __fdiv_rn(-127.0f, vmax);
#pragma unroll
        for (int i = 0; i < 8; ++i) q[i] = min(127, __float2int_rn(iscale * v[i]));
        d = __fdiv_rn(1.0f, iscale);
    } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) q[i] = 0;
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int k = half * 128 + 4 * lane;
        const int * qq = q + 4 * half;
        *(uint32_t *)(rec + k0 + k) = (uint32_t)(qq[0] & 0xFF) | ((uint32_t)(qq[1] & 0xFF) << 8) | ((uint32_t)(qq[2] & 0xFF) << 16) | ((uint32_t)(qq[3] & 0xFF) << 24);
        int s = qq[0] + qq[1] + qq[2] + qq[3];
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        if ((lane & 3) == 0) *(int16_t *)(rec + L.off_bs + ((k0 + k) >> 4) * 2) = (int16_t)s;
    }
    if (lane == 0) ((float *)(rec + L.off_d))[k0 >> 8] = d;
}

// all warps of the CTA quantize one activation row x[0..K) into `rec` (shared or global)
template <bool KQ> __device__ __forceinline__ void cta_quantize_row(const float * x, int64_t K, uint8_t * rec, const act_layout & L) {
    const int warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    for (int64_t k0 = (int64_t)warp * 256; k0 < K; k0 += (int64_t)nwarp * 256) {
        if constexpr (KQ) warp_quantize_q8_K_x256(x + k0, rec, L, (int)k0);
        else              warp_quantize_q8_0_x256(x + k0, (int)min((int64_t)256, K - k0), rec, L, (int)k0);
    }
}

} // namespace b200
