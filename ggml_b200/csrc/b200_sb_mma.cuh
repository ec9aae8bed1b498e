// b200_sb_mma.cuh — small-batch consume path of the bandwidth mat-vec kernel on the int8 tensor-core instruction
// `mma.sync.aligned.m16n8k32.s32.s8.s8.s32`: one warp multiplies a tile of 16 weight rows x 32 weights with 8 activation columns.
//
// Why: with 2..8 activation columns the dp4a task dots of b200_sb_tasks.cuh are issue-bound — a
// lane decodes its 256 weights once and then pays one dp4a per 4 weights per COLUMN, and every column's int8 record is re-read from
// shared memory per row.  Here a warp's 32 lanes hold the 16 x 32 weight fragment and the 32 x 8 activation fragment of one
// sub-block, so eight columns cost the instructions of one, the activations are read once per 16 rows, and the arithmetic stays the
// reference's: integer dot products of the same int8 codes (ggml-cpu's quantize_row_q8_0 / q8_K), f32 scaling per block.
//
// Fragment layout (PTX ISA, m16n8k32 .s8): lane = 4 g + t.  A: a0 = row g, k-slots 4t..4t+3; a1 = row g+8, same slots; a2 / a3 = the
// same rows, slots 16+4t..  B: b0 = column g, slots 4t..; b1 = slots 16+4t..  D: c0 = (row g, col 2t), c1 = (g, 2t+1), c2 = (g+8, 2t),
// c3 = (g+8, 2t+1).  The sum over k is order-free, so slot s of lane t is mapped to weight / activation index 8t + (s & 3) + 4 (s >> 4)
// of the sub-block: every lane then fetches its slots with ONE 8-byte load from the packed weights and one from the int8 activations.
//
// Pure per-thread code (plus the mma), compiled for the host by tests/hostemu (the mma becomes an exchange between 32 lockstep threads).
#pragma once
#include "b200_sb_tasks.cuh"

namespace b200 {

// ----------------------------------------------------------------------------- planar activation records (one per column)
//   +0        q   : K int8 codes in natural order
//   +off_h32  h32 : per 32-value block one int16 sum of its codes (16 bytes per 256-value task)
//   +off_s16  s16 : (formats with 16-wide scale groups) per 16 values one int16 sum (32 bytes per task); absent otherwise
//   +off_d    d   : Q8_K family: one float per task; Q8_0 family: one float per 32-value block (fp16-rounded)
//   +off_s    s   : (weight formats with a minimum, Q4_1 / Q5_1) block_q8_1.s = fp16(d_unrounded * sum of the block's codes), as a float per block
// col_bytes = 32 (mod 128): the eight columns' 8-byte fragment loads of a half-warp fall into distinct bank groups (formats whose lanes
// load 4-byte fragments, Q6_K: 16 (mod 128), eight columns x 16 bytes = all 32 banks).
struct mma_act {
    int32_t ntask, off_h32, off_s16, off_d, off_s, col_bytes;
};
__host__ __device__ inline mma_act make_mma_act(int64_t K, bool kq, bool s16, int residue = 32, bool s81 = false) {
    mma_act A;
    A.ntask = (int32_t)(K / 256);
    A.off_h32 = (int32_t)K;
    A.off_s16 = A.off_h32 + 16 * A.ntask;
    A.off_d = A.off_s16 + (s16 ? 32 * A.ntask : 0);
    A.off_s = A.off_d + (kq ? 4 : 32) * A.ntask;
    int32_t bytes = A.off_s + (s81 ? 32 * A.ntask : 0);
    bytes = (bytes + 15) & ~15;
    while ((bytes & 127) != residue) bytes += 16;
    A.col_bytes = bytes;
    return A;
}

// half a warp quantizes act-task t of one column into the planar record at `col` (same arithmetic as sb_quantize_task_h)
template <bool KQ, bool S16, bool S81 = false> __device__ __forceinline__ void mma_quantize_task_h(const float * __restrict__ x, bool valid, uint8_t * col, const mma_act & A, int t) {
    const int l = threadIdx.x & 15;
    const sb_qtask r = sb_quantize_core<KQ>(x, valid, t);
    if (valid) {
        *(int4 *)(col + 256 * t + 16 * l) = r.pk;
        if constexpr (S16) *(int16_t *)(col + A.off_s16 + 32 * t + 2 * l) = (int16_t)r.s;
        if ((l & 1) == 0) *(int16_t *)(col + A.off_h32 + 16 * t + 2 * (l >> 1)) = (int16_t)r.s2;
        if constexpr (KQ) { if (l == 0) *(float *)(col + A.off_d + 4 * t) = r.d; }
        else              { if ((l & 1) == 0) *(float *)(col + A.off_d + 32 * t + 4 * (l >> 1)) = r.d; }
        if constexpr (!KQ && S81) { if ((l & 1) == 0) *(float *)(col + A.off_s + 32 * t + 4 * (l >> 1)) = __half2float(__float2half_rn(__fmul_rn(r.dun, (float)r.s2))); }
    }
}

// ----------------------------------------------------------------------------- the instruction
#ifndef B200_HOST_EMU
__device__ __forceinline__ void mma_s8_16x8x32(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
                 : "=r"(c[0]), "=r"(c[1]), "=r"(c[2]), "=r"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "r"(0));
}
// A bytes unsigned (0..255): high nibbles used in place (q & 0xF0 = 16 x the nibble; the result is an exact multiple of 16)
__device__ __forceinline__ void mma_u8s8_16x8x32(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
                 : "=r"(c[0]), "=r"(c[1]), "=r"(c[2]), "=r"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "r"(0));
}
// 8 bytes at an address whose residue mod 8 is the compile-time constant R (block formats are only 2-byte aligned): aligned loads + funnel shifts
template <int R> __device__ __forceinline__ uint2 lds8(const uint8_t * p) {
    static_assert(R == 0 || R == 2 || R == 4 || R == 6, "two-byte aligned");
    if constexpr (R == 0) return *(const uint2 *)p;
    else if constexpr (R == 4) { uint2 v; v.x = *(const uint32_t *)p; v.y = *(const uint32_t *)(p + 4); return v; }
    else if constexpr (R == 2) {
        const uint2 lo = *(const uint2 *)(p - 2); const uint32_t hi = *(const uint32_t *)(p + 6);
        uint2 v; v.x = __funnelshift_r(lo.x, lo.y, 16); v.y = __funnelshift_r(lo.y, hi, 16); return v;
    } else {
        const uint32_t lo = *(const uint32_t *)(p - 2); const uint2 hi = *(const uint2 *)(p + 2);
        uint2 v; v.x = __funnelshift_r(lo, hi.x, 16); v.y = __funnelshift_r(hi.x, hi.y, 16); return v;
    }
}
__device__ __forceinline__ uint32_t lds_u16(const uint8_t * p) { return *(const uint16_t *)p; }
// m16n8k16: lane 4g+t holds A (row g, k 4t..4t+3), (row g+8, same k) and B (k 4t..4t+3, column g); D as m16n8k32
__device__ __forceinline__ void mma_s8_16x8x16(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t b0) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%7,%7,%7,%7};"
                 : "=r"(c[0]), "=r"(c[1]), "=r"(c[2]), "=r"(c[3]) : "r"(a0), "r"(a1), "r"(b0), "r"(0));
}
// a 32-bit word at an address whose residue mod 4 is the compile-time constant R (0 or 2)
template <int R> __device__ __forceinline__ uint32_t lds4(const uint8_t * p) {
    if constexpr (R == 0) return *(const uint32_t *)p;
    else return __funnelshift_r(*(const uint32_t *)(p - 2), *(const uint32_t *)(p + 2), 16);
}
#else
// host restatement: every lane publishes its fragments, then computes its four outputs from all lanes' fragments
template <bool A_UNSIGNED>
inline void mma_emu_16x8x32(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    static uint32_t fr[32][6];
    const int lane = (int)(threadIdx.x & 31);
    fr[lane][0] = a0; fr[lane][1] = a1; fr[lane][2] = a2; fr[lane][3] = a3; fr[lane][4] = b0; fr[lane][5] = b1;
    pthread_barrier_wait(&warp_emu::barrier());
    const int g = lane >> 2, t = lane & 3;
    for (int i = 0; i < 4; ++i) {
        const int row = g + 8 * (i >> 1), coln = 2 * t + (i & 1);
        int sum = 0;
        for (int tt = 0; tt < 4; ++tt) {
            const uint32_t * A = fr[4 * (row & 7) + tt], * B = fr[4 * coln + tt];
            const uint32_t alo = A[row >> 3], ahi = A[2 + (row >> 3)];
            if (A_UNSIGNED) { sum = dp4a_us(alo, (int)B[4], sum); sum = dp4a_us(ahi, (int)B[5], sum); }
            else            { sum = __dp4a((int)alo, (int)B[4], sum); sum = __dp4a((int)ahi, (int)B[5], sum); }
        }
        c[i] = sum;
    }
    pthread_barrier_wait(&warp_emu::barrier());
}
inline void mma_s8_16x8x32(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) { mma_emu_16x8x32<false>(c, a0, a1, a2, a3, b0, b1); }
inline void mma_u8s8_16x8x32(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) { mma_emu_16x8x32<true>(c, a0, a1, a2, a3, b0, b1); }
inline void mma_s8_16x8x16(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t b0) {
    static uint32_t fr[32][3];
    const int lane = (int)(threadIdx.x & 31);
    fr[lane][0] = a0; fr[lane][1] = a1; fr[lane][2] = b0;
    pthread_barrier_wait(&warp_emu::barrier());
    const int g = lane >> 2, t = lane & 3;
    for (int i = 0; i < 4; ++i) {
        const int row = g + 8 * (i >> 1), coln = 2 * t + (i & 1);
        int sum = 0;
        for (int tt = 0; tt < 4; ++tt) sum = __dp4a((int)fr[4 * (row & 7) + tt][row >> 3], (int)fr[4 * coln + tt][2], sum);
        c[i] = sum;
    }
    pthread_barrier_wait(&warp_emu::barrier());
}
template <int R> inline uint32_t lds4(const uint8_t * p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
template <int R> inline uint2 lds8(const uint8_t * p) { uint2 v; std::memcpy(&v, p, 8); return v; }
inline uint32_t lds_u16(const uint8_t * p) { uint16_t v; std::memcpy(&v, p, 2); return v; }
#endif

// sixteen bytes at a 4-byte aligned address
__device__ __forceinline__ int4 lds128w(const uint8_t * p) {
    const uint32_t * q = (const uint32_t *)p;
    int4 v; v.x = (int)q[0]; v.y = (int)q[1]; v.z = (int)q[2]; v.w = (int)q[3];
    return v;
}

// what a lane needs of the activation columns for one task: its B column (fragment loads) and its two output columns (sums, scales)
struct mma_cols {
    const uint8_t * b;       // column g (clamped to the last real column): B fragments
    const uint8_t * c0, * c1;   // columns 2t and 2t+1 (clamped): h32 / s16 / d of the outputs this lane accumulates
};

// bytes of a 256-weight task in the packed row
template <int T> struct mmafmt;
// RESIDUE: row pitch of the weight stage and column pitch of the records mod 128 (lanes load 8-byte fragments: 32; 4-byte fragments: 16)
template <> struct mmafmt<T_Q4_K> { static constexpr int TASK_B = 144, RESIDUE = 32; static constexpr bool KQ = true,  S16 = false; };
template <> struct mmafmt<T_Q5_K> { static constexpr int TASK_B = 176, RESIDUE = 32; static constexpr bool KQ = true,  S16 = false; };
template <> struct mmafmt<T_Q4_0> { static constexpr int TASK_B = 144, RESIDUE = 32; static constexpr bool KQ = false, S16 = false; };
template <> struct mmafmt<T_Q8_0> { static constexpr int TASK_B = 272, RESIDUE = 32; static constexpr bool KQ = false, S16 = false; };
template <> struct mmafmt<T_Q6_K> { static constexpr int TASK_B = 210, RESIDUE = 16; static constexpr bool KQ = true,  S16 = true;  };
template <> struct mmafmt<T_Q5_0>   { static constexpr int TASK_B = 176, RESIDUE = 32; static constexpr bool KQ = false, S16 = false; };
template <> struct mmafmt<T_Q4_1>   { static constexpr int TASK_B = 160, RESIDUE = 32; static constexpr bool KQ = false, S16 = false, S81 = true; };
template <> struct mmafmt<T_Q5_1>   { static constexpr int TASK_B = 192, RESIDUE = 32; static constexpr bool KQ = false, S16 = false, S81 = true; };
template <> struct mmafmt<T_IQ4_NL> { static constexpr int TASK_B = 144, RESIDUE = 32; static constexpr bool KQ = false, S16 = false; };
template <> struct mmafmt<T_IQ4_XS> { static constexpr int TASK_B = 136, RESIDUE = 32; static constexpr bool KQ = true,  S16 = false; };
template <> struct mmafmt<T_Q2_K>   { static constexpr int TASK_B = 84,  RESIDUE = 16; static constexpr bool KQ = true,  S16 = true;  };
template <> struct mmafmt<T_Q3_K>   { static constexpr int TASK_B = 110, RESIDUE = 16; static constexpr bool KQ = true,  S16 = true;  };
// (formats without a minimum: no Q8_1 s region)
template <int T, typename = void> struct mma_s81 { static constexpr bool value = false; };
template <int T> struct mma_s81<T, decltype((void)mmafmt<T>::S81)> { static constexpr bool value = mmafmt<T>::S81; };

// One task (256 weights) of rows g (w0) and g+8 (w1) against the eight columns: facc[i] += the task's contribution to output i of the
// D fragment.  `task` = index of the task in the row (selects the activation slice), t = lane & 3.
template <int T> __device__ __forceinline__ void mma_task(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]);

template <bool FIVE>
__device__ __forceinline__ void mma_q45_task(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) {
    const int4 hA = lds128(w0), hB = lds128(w1);                    // d | dmin | scales[12] of the two rows
    // the 6-bit (scale, min) pairs of get_scale_min_k4, four sub-blocks per word (as q45_task)
    const uint32_t scA[2] = { (uint32_t)hA.y & 0x3F3F3F3Fu, ((uint32_t)hA.w & 0x0F0F0F0Fu) | (((uint32_t)hA.y >> 2) & 0x30303030u) };
    const uint32_t mnA[2] = { (uint32_t)hA.z & 0x3F3F3F3Fu, (((uint32_t)hA.w >> 4) & 0x0F0F0F0Fu) | (((uint32_t)hA.z >> 2) & 0x30303030u) };
    const uint32_t scB[2] = { (uint32_t)hB.y & 0x3F3F3F3Fu, ((uint32_t)hB.w & 0x0F0F0F0Fu) | (((uint32_t)hB.y >> 2) & 0x30303030u) };
    const uint32_t mnB[2] = { (uint32_t)hB.z & 0x3F3F3F3Fu, (((uint32_t)hB.w >> 4) & 0x0F0F0F0Fu) | (((uint32_t)hB.z >> 2) & 0x30303030u) };
    uint2 qhA = { 0, 0 }, qhB = { 0, 0 };
    if constexpr (FIVE) { qhA = *(const uint2 *)(w0 + 16 + 8 * t); qhB = *(const uint2 *)(w1 + 16 + 8 * t); }   // bit j of byte i = high bit of weight i of sub-block j
    const uint8_t * qa = w0 + (FIVE ? 48 : 16) + 8 * t, * qb = w1 + (FIVE ? 48 : 16) + 8 * t;
    const uint8_t * y = C.b + 256 * task + 8 * t;
    int acc[4] = { 0, 0, 0, 0 }, acc16[4] = { 0, 0, 0, 0 };         // acc16: sums of the in-place high nibbles (16 x the nibble dot), Q4_K only
#pragma unroll
    for (int p = 0; p < 4; ++p) {                                   // 64 weights: sub-block 2p in the low nibbles, 2p+1 in the high ones
        const uint2 wa = *(const uint2 *)(qa + 32 * p), wb = *(const uint2 *)(qb + 32 * p);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int j = 2 * p + h;
            const uint2 yy = *(const uint2 *)(y + 32 * j);
            const int sa = (j & 3) == 0 ? ubyte<0>(scA[j >> 2]) : (j & 3) == 1 ? ubyte<1>(scA[j >> 2]) : (j & 3) == 2 ? ubyte<2>(scA[j >> 2]) : ubyte<3>(scA[j >> 2]);
            const int sb = (j & 3) == 0 ? ubyte<0>(scB[j >> 2]) : (j & 3) == 1 ? ubyte<1>(scB[j >> 2]) : (j & 3) == 2 ? ubyte<2>(scB[j >> 2]) : ubyte<3>(scB[j >> 2]);
            int c[4];
            if constexpr (!FIVE) {
                if (h == 0) {
                    mma_s8_16x8x32(c, wa.x & 0x0F0F0F0Fu, wb.x & 0x0F0F0F0Fu, wa.y & 0x0F0F0F0Fu, wb.y & 0x0F0F0F0Fu, yy.x, yy.y);
                    acc[0] += sa * c[0]; acc[1] += sa * c[1]; acc[2] += sb * c[2]; acc[3] += sb * c[3];
                } else {
                    mma_u8s8_16x8x32(c, wa.x & 0xF0F0F0F0u, wb.x & 0xF0F0F0F0u, wa.y & 0xF0F0F0F0u, wb.y & 0xF0F0F0F0u, yy.x, yy.y);
                    acc16[0] += sa * c[0]; acc16[1] += sa * c[1]; acc16[2] += sb * c[2]; acc16[3] += sb * c[3];
                }
            } else {
                const uint32_t a0 = ((wa.x >> (4 * h)) & 0x0F0F0F0Fu) | (((qhA.x >> j) & 0x01010101u) << 4), a2 = ((wa.y >> (4 * h)) & 0x0F0F0F0Fu) | (((qhA.y >> j) & 0x01010101u) << 4);
                const uint32_t a1 = ((wb.x >> (4 * h)) & 0x0F0F0F0Fu) | (((qhB.x >> j) & 0x01010101u) << 4), a3 = ((wb.y >> (4 * h)) & 0x0F0F0F0Fu) | (((qhB.y >> j) & 0x01010101u) << 4);
                mma_s8_16x8x32(c, a0, a1, a2, a3, yy.x, yy.y);
                acc[0] += sa * c[0]; acc[1] += sa * c[1]; acc[2] += sb * c[2]; acc[3] += sb * c[3];
            }
        }
    }
    if constexpr (!FIVE) {
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] += acc16[i] >> 4;        // exact: every term is a multiple of 16
    }
    // mins: sum_j min_j(row) * (sum of the 32 activations of sub-block j)(column), two sub-blocks per dp2a
    const int4 s0 = lds128(C.c0 + A.off_h32 + 16 * task), s1 = lds128(C.c1 + A.off_h32 + 16 * task);
    auto mins = [](const int4 & s, const uint32_t (&mn)[2]) {
        int m = dp2a_lo_su(s.x, mn[0], 0);
        m = dp2a_hi_su(s.y, mn[0], m);
        m = dp2a_lo_su(s.z, mn[1], m);
        return dp2a_hi_su(s.w, mn[1], m);
    };
    const float yd0 = *(const float *)(C.c0 + A.off_d + 4 * task), yd1 = *(const float *)(C.c1 + A.off_d + 4 * task);
    const float dA = h2f((uint32_t)hA.x & 0xFFFF), mA = h2f((uint32_t)hA.x >> 16), dB = h2f((uint32_t)hB.x & 0xFFFF), mB = h2f((uint32_t)hB.x >> 16);
    facc[0] += (dA * yd0) * (float)acc[0] - (mA * yd0) * (float)mins(s0, mnA);
    facc[1] += (dA * yd1) * (float)acc[1] - (mA * yd1) * (float)mins(s1, mnA);
    facc[2] += (dB * yd0) * (float)acc[2] - (mB * yd0) * (float)mins(s0, mnB);
    facc[3] += (dB * yd1) * (float)acc[3] - (mB * yd1) * (float)mins(s1, mnB);
}
template <> __device__ __forceinline__ void mma_task<T_Q4_K>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) { mma_q45_task<false>(w0, w1, C, A, task, t, facc); }
template <> __device__ __forceinline__ void mma_task<T_Q5_K>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) { mma_q45_task<true>(w0, w1, C, A, task, t, facc); }

// 32-weight block formats: a task = eight blocks.  Block layouts (bytes): Q4_0 / IQ4_NL d | qs[16]; Q5_0 d | qh[4] | qs[16]; Q4_1 d | m | qs[16];
// Q5_1 d | m | qh[4] | qs[16]; Q8_0 d | int8[32].  4-bit formats: weight i in the low nibble of qs[i], weight i + 16 in the high one, fifth bit i of qh.
// Block b starts at BLK * b from a 16-byte aligned task base: the residue of every fragment load mod 8 (mod 4) is a compile-time constant.
template <int T> struct blk32fmt;
template <> struct blk32fmt<T_Q4_0>   { static constexpr int BLK = 18, QS = 2, QH = -1, OFF = 8;  static constexpr bool NIB = true,  MIN = false, LUT = false; };
template <> struct blk32fmt<T_IQ4_NL> { static constexpr int BLK = 18, QS = 2, QH = -1, OFF = 0;  static constexpr bool NIB = true,  MIN = false, LUT = true;  };
template <> struct blk32fmt<T_Q5_0>   { static constexpr int BLK = 22, QS = 6, QH = 2,  OFF = 16; static constexpr bool NIB = true,  MIN = false, LUT = false; };
template <> struct blk32fmt<T_Q4_1>   { static constexpr int BLK = 20, QS = 4, QH = -1, OFF = 0;  static constexpr bool NIB = true,  MIN = true,  LUT = false; };
template <> struct blk32fmt<T_Q5_1>   { static constexpr int BLK = 24, QS = 8, QH = 4,  OFF = 0;  static constexpr bool NIB = true,  MIN = true,  LUT = false; };
template <> struct blk32fmt<T_Q8_0>   { static constexpr int BLK = 34, QS = 2, QH = -1, OFF = 0;  static constexpr bool NIB = false, MIN = false, LUT = false; };

template <int T, int B>
__device__ __forceinline__ void mma_blk32(const uint8_t * w0, const uint8_t * w1, const uint8_t * y, const int4 & s0, const int4 & s1,
                                         const float (&yd0)[8], const float (&yd1)[8], const float (&ys0)[8], const float (&ys1)[8], int t, float (&facc)[4]) {
    using F = blk32fmt<T>;
    constexpr int BLK = F::BLK, R = (BLK * B + F::QS) & 7;
    const int off = BLK * B + F::QS + (F::NIB ? 8 * (t & 1) : 8 * t);
    const uint2 wa = lds8<R>(w0 + off), wb = lds8<R>(w1 + off);
    const uint2 yy = *(const uint2 *)(y + 32 * B);
    uint32_t a0 = wa.x, a2 = wa.y, a1 = wb.x, a3 = wb.y;
    if constexpr (F::NIB) {                                         // lanes t = 0, 1 hold weights 0..15 (low nibbles), t = 2, 3 weights 16..31 (high nibbles)
        const int sh = (t >> 1) * 4;
        a0 = (a0 >> sh) & 0x0F0F0F0Fu; a2 = (a2 >> sh) & 0x0F0F0F0Fu; a1 = (a1 >> sh) & 0x0F0F0F0Fu; a3 = (a3 >> sh) & 0x0F0F0F0Fu;
    }
    if constexpr (F::QH >= 0) {                                     // fifth bits 8t .. 8t+7 of the block's 32
        constexpr int RH = (BLK * B + F::QH) & 3;
        const uint32_t ha = (lds4<RH>(w0 + BLK * B + F::QH) >> (8 * t)) & 0xFFu, hb = (lds4<RH>(w1 + BLK * B + F::QH) >> (8 * t)) & 0xFFu;
        a0 |= spread4_to_bit4(ha); a2 |= spread4_to_bit4(ha >> 4); a1 |= spread4_to_bit4(hb); a3 |= spread4_to_bit4(hb >> 4);
    }
    if constexpr (F::LUT) { a0 = iq4nl_lookup4(a0); a1 = iq4nl_lookup4(a1); a2 = iq4nl_lookup4(a2); a3 = iq4nl_lookup4(a3); }
    int c[4];
    mma_s8_16x8x32(c, a0, a1, a2, a3, yy.x, yy.y);
    const float dA = h2f(lds_u16(w0 + BLK * B)), dB = h2f(lds_u16(w1 + BLK * B));
    if constexpr (F::OFF != 0) {                                    // codes are q - OFF: subtract OFF x (sum of the block's activations)
        const int * p0 = &s0.x, * p1 = &s1.x;
        const int h0 = (B & 1) ? (p0[B >> 1] >> 16) : (int)(int16_t)(p0[B >> 1] & 0xFFFF);
        const int h1 = (B & 1) ? (p1[B >> 1] >> 16) : (int)(int16_t)(p1[B >> 1] & 0xFFFF);
        c[0] -= F::OFF * h0; c[1] -= F::OFF * h1; c[2] -= F::OFF * h0; c[3] -= F::OFF * h1;
    }
    if constexpr (T == T_Q4_0) {
        facc[0] += (float)c[0] * dA * yd0[B]; facc[1] += (float)c[1] * dA * yd1[B];
        facc[2] += (float)c[2] * dB * yd0[B]; facc[3] += (float)c[3] * dB * yd1[B];
    } else if constexpr (T == T_Q8_0) {
        facc[0] += (float)c[0] * (dA * yd0[B]); facc[1] += (float)c[1] * (dA * yd1[B]);
        facc[2] += (float)c[2] * (dB * yd0[B]); facc[3] += (float)c[3] * (dB * yd1[B]);
    } else if constexpr (F::MIN) {
        const float mA = h2f(lds_u16(w0 + BLK * B + 2)), mB = h2f(lds_u16(w1 + BLK * B + 2));
        facc[0] += (dA * yd0[B]) * (float)c[0] + mA * ys0[B]; facc[1] += (dA * yd1[B]) * (float)c[1] + mA * ys1[B];
        facc[2] += (dB * yd0[B]) * (float)c[2] + mB * ys0[B]; facc[3] += (dB * yd1[B]) * (float)c[3] + mB * ys1[B];
    } else {
        facc[0] += (dA * yd0[B]) * (float)c[0]; facc[1] += (dA * yd1[B]) * (float)c[1];
        facc[2] += (dB * yd0[B]) * (float)c[2]; facc[3] += (dB * yd1[B]) * (float)c[3];
    }
}
__device__ __forceinline__ void mma_load8f(const uint8_t * p, float (&v)[8]) {
    const int4 a = lds128(p), b = lds128(p + 16);
    v[0] = __int_as_float(a.x); v[1] = __int_as_float(a.y); v[2] = __int_as_float(a.z); v[3] = __int_as_float(a.w);
    v[4] = __int_as_float(b.x); v[5] = __int_as_float(b.y); v[6] = __int_as_float(b.z); v[7] = __int_as_float(b.w);
}
template <int T>
__device__ __forceinline__ void mma_blk32_task(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) {
    using F = blk32fmt<T>;
    const uint8_t * y = C.b + 256 * task + 8 * t;
    int4 s0 = { 0, 0, 0, 0 }, s1 = { 0, 0, 0, 0 };
    if constexpr (F::OFF != 0) { s0 = lds128(C.c0 + A.off_h32 + 16 * task); s1 = lds128(C.c1 + A.off_h32 + 16 * task); }
    float yd0[8], yd1[8], ys0[8] = { 0, 0, 0, 0, 0, 0, 0, 0 }, ys1[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    mma_load8f(C.c0 + A.off_d + 32 * task, yd0); mma_load8f(C.c1 + A.off_d + 32 * task, yd1);
    if constexpr (F::MIN) { mma_load8f(C.c0 + A.off_s + 32 * task, ys0); mma_load8f(C.c1 + A.off_s + 32 * task, ys1); }
    mma_blk32<T, 0>(w0, w1, y, s0, s1, yd0, yd1, ys0, ys1, t, facc); mma_blk32<T, 1>(w0, w1, y, s0, s1, yd0, yd1, ys0, ys1, t, facc);
    mma_blk32<T, 2>(w0, w1, y, s0, s1, yd0, yd1, ys0, ys1, t, facc); mma_blk32<T, 3>(w0, w1, y, s0, s1, yd0, yd1, ys0, ys1, t, facc);
    mma_blk32<T, 4>(w0, w1, y, s0, s1, yd0, yd1, ys0, ys1, t, facc); mma_blk32<T, 5>(w0, w1, y, s0, s1, yd0, yd1, ys0, ys1, t, facc);
    mma_blk32<T, 6>(w0, w1, y, s0, s1, yd0, yd1, ys0, ys1, t, facc); mma_blk32<T, 7>(w0, w1, y, s0, s1, yd0, yd1, ys0, ys1, t, facc);
}
template <> __device__ __forceinline__ void mma_task<T_Q4_0>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) { mma_blk32_task<T_Q4_0>(w0, w1, C, A, task, t, facc); }
template <> __device__ __forceinline__ void mma_task<T_Q8_0>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) { mma_blk32_task<T_Q8_0>(w0, w1, C, A, task, t, facc); }
template <> __device__ __forceinline__ void mma_task<T_Q5_0>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) { mma_blk32_task<T_Q5_0>(w0, w1, C, A, task, t, facc); }
template <> __device__ __forceinline__ void mma_task<T_Q4_1>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) { mma_blk32_task<T_Q4_1>(w0, w1, C, A, task, t, facc); }
template <> __device__ __forceinline__ void mma_task<T_Q5_1>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) { mma_blk32_task<T_Q5_1>(w0, w1, C, A, task, t, facc); }
template <> __device__ __forceinline__ void mma_task<T_IQ4_NL>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) { mma_blk32_task<T_IQ4_NL>(w0, w1, C, A, task, t, facc); }

// IQ4_XS: 136-byte superblocks (d | scales_h | scales_l[4] | qs[128]), eight 32-weight sub-blocks laid out as Q4_0 blocks (weight i in the low nibble
// of qs[16 ib + i], weight i + 16 in the high one), nibbles mapped through the IQ4_NL codebook, 6-bit sub-block scales (value - 32), Q8_K activations.
template <> __device__ __forceinline__ void mma_task<T_IQ4_XS>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) {
    const uint2 hA = *(const uint2 *)w0, hB = *(const uint2 *)w1;
    const uint8_t * y = C.b + 256 * task + 8 * t;
    const int sh = (t >> 1) * 4;
    int acc[4] = { 0, 0, 0, 0 };
#pragma unroll
    for (int ib = 0; ib < 8; ++ib) {
        const uint2 wa = *(const uint2 *)(w0 + 8 + 16 * ib + 8 * (t & 1)), wb = *(const uint2 *)(w1 + 8 + 16 * ib + 8 * (t & 1));
        const uint2 yy = *(const uint2 *)(y + 32 * ib);
        int c[4];
        mma_s8_16x8x32(c, iq4nl_lookup4((wa.x >> sh) & 0x0F0F0F0Fu), iq4nl_lookup4((wb.x >> sh) & 0x0F0F0F0Fu),
                          iq4nl_lookup4((wa.y >> sh) & 0x0F0F0F0Fu), iq4nl_lookup4((wb.y >> sh) & 0x0F0F0F0Fu), yy.x, yy.y);
        const int sa = iq4xs_scale(hA.x, hA.y, ib), sb = iq4xs_scale(hB.x, hB.y, ib);
        acc[0] += sa * c[0]; acc[1] += sa * c[1]; acc[2] += sb * c[2]; acc[3] += sb * c[3];
    }
    const float yd0 = *(const float *)(C.c0 + A.off_d + 4 * task), yd1 = *(const float *)(C.c1 + A.off_d + 4 * task);
    const float dA = h2f(hA.x & 0xFFFF), dB = h2f(hB.x & 0xFFFF);
    facc[0] += (dA * yd0) * (float)acc[0]; facc[1] += (dA * yd1) * (float)acc[1];
    facc[2] += (dB * yd0) * (float)acc[2]; facc[3] += (dB * yd1) * (float)acc[3];
}

// Q2_K: 84-byte superblocks (scales[16]: 4-bit scale | 4-bit min << 4, qs[64], d | dmin), sixteen 16-weight groups -> sixteen m16n8k16 products.
// Group g = 8 h + 2 jj + half: weights 16 g .. 16 g + 15 = bits 2 jj, 2 jj + 1 of qs[32 h + 16 half .. + 15].
template <> __device__ __forceinline__ void mma_task<T_Q2_K>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) {
    const int4 sA = lds128w(w0), sB = lds128w(w1);                  // the sixteen scale bytes of the two rows (4-byte aligned superblocks: four word loads)
    const uint32_t scA[4] = { (uint32_t)sA.x, (uint32_t)sA.y, (uint32_t)sA.z, (uint32_t)sA.w }, scB[4] = { (uint32_t)sB.x, (uint32_t)sB.y, (uint32_t)sB.z, (uint32_t)sB.w };
    const uint8_t * y = C.b + 256 * task + 4 * t;
    int acc[4] = { 0, 0, 0, 0 };
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const uint32_t qa = *(const uint32_t *)(w0 + 16 + 32 * h + 16 * half + 4 * t), qb = *(const uint32_t *)(w1 + 16 + 32 * h + 16 * half + 4 * t);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                const int g = 8 * h + 2 * jj + half;                // compile time
                const uint32_t b0 = *(const uint32_t *)(y + 16 * g);
                int c[4];
                mma_s8_16x8x16(c, (qa >> (2 * jj)) & 0x03030303u, (qb >> (2 * jj)) & 0x03030303u, b0);
                const uint32_t wa = scA[g >> 2] & 0x0F0F0F0Fu, wb = scB[g >> 2] & 0x0F0F0F0Fu;
                const int sa = (g & 3) == 0 ? ubyte<0>(wa) : (g & 3) == 1 ? ubyte<1>(wa) : (g & 3) == 2 ? ubyte<2>(wa) : ubyte<3>(wa);
                const int sb = (g & 3) == 0 ? ubyte<0>(wb) : (g & 3) == 1 ? ubyte<1>(wb) : (g & 3) == 2 ? ubyte<2>(wb) : ubyte<3>(wb);
                acc[0] += sa * c[0]; acc[1] += sa * c[1]; acc[2] += sb * c[2]; acc[3] += sb * c[3];
            }
        }
    }
    // mins: sum over the sixteen groups of min_g x (16-sum of the column's activations)
    auto mins = [](const int4 & sa, const int4 & sb, const uint32_t (&sc)[4]) {
        const uint32_t m0 = (sc[0] >> 4) & 0x0F0F0F0Fu, m1 = (sc[1] >> 4) & 0x0F0F0F0Fu, m2 = (sc[2] >> 4) & 0x0F0F0F0Fu, m3 = (sc[3] >> 4) & 0x0F0F0F0Fu;
        int m = dp2a_lo_su(sa.x, m0, 0);
        m = dp2a_hi_su(sa.y, m0, m); m = dp2a_lo_su(sa.z, m1, m); m = dp2a_hi_su(sa.w, m1, m);
        m = dp2a_lo_su(sb.x, m2, m); m = dp2a_hi_su(sb.y, m2, m); m = dp2a_lo_su(sb.z, m3, m);
        return dp2a_hi_su(sb.w, m3, m);
    };
    const int4 s0a = lds128(C.c0 + A.off_s16 + 32 * task), s0b = lds128(C.c0 + A.off_s16 + 32 * task + 16);
    const int4 s1a = lds128(C.c1 + A.off_s16 + 32 * task), s1b = lds128(C.c1 + A.off_s16 + 32 * task + 16);
    const float yd0 = *(const float *)(C.c0 + A.off_d + 4 * task), yd1 = *(const float *)(C.c1 + A.off_d + 4 * task);
    const uint32_t ddA = *(const uint32_t *)(w0 + 80), ddB = *(const uint32_t *)(w1 + 80);
    const float dA = h2f(ddA & 0xFFFF), mA = h2f(ddA >> 16), dB = h2f(ddB & 0xFFFF), mB = h2f(ddB >> 16);
    facc[0] += (yd0 * dA) * (float)acc[0] - (yd0 * mA) * (float)mins(s0a, s0b, scA);
    facc[1] += (yd1 * dA) * (float)acc[1] - (yd1 * mA) * (float)mins(s1a, s1b, scA);
    facc[2] += (yd0 * dB) * (float)acc[2] - (yd0 * mB) * (float)mins(s0a, s0b, scB);
    facc[3] += (yd1 * dB) * (float)acc[3] - (yd1 * mB) * (float)mins(s1a, s1b, scB);
}

// Q3_K: 110-byte superblocks (hmask[32] | qs[64] | scales[12] | d), 2-byte aligned like Q6_K; sixteen 16-weight groups -> sixteen m16n8k16 products.
// Group g = 8 h + 2 jj + half: bits 2 jj, 2 jj + 1 of qs[32 h + 16 half .. + 15] plus bit (4 h + jj) of hmask[16 half .. + 15] as bit 2; value = code - 4
// (the "- 4" is sum_g scale_g * 4 * (16-sum of the activations)_g); scales are 6 bits (value - 32), low nibbles in bytes 0..7, high bits in bytes 8..11.
template <int R>
__device__ __forceinline__ void mma_q3_task(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) {
    auto scales = [](const uint8_t * w, uint32_t (&sc)[4]) {
        const uint32_t s0 = lds4<R>(w + 96), s1 = lds4<R>(w + 100), s2 = lds4<R>(w + 104);
        const uint32_t aux[4] = { ( s0       & 0x0F0F0F0Fu) | (( s2       & 0x03030303u) << 4), ( s1       & 0x0F0F0F0Fu) | (((s2 >> 2) & 0x03030303u) << 4),
                                  ((s0 >> 4) & 0x0F0F0F0Fu) | (((s2 >> 4) & 0x03030303u) << 4), ((s1 >> 4) & 0x0F0F0F0Fu) | (((s2 >> 6) & 0x03030303u) << 4) };
#pragma unroll
        for (int i = 0; i < 4; ++i) {                               // 6-bit x -> int8 (x - 32): flip bit 5, then replicate it into bits 6 and 7
            const uint32_t y = aux[i] ^ 0x20202020u, m = y & 0x20202020u;
            sc[i] = y | (m << 1) | (m << 2);
        }
    };
    uint32_t scA[4], scB[4];
    scales(w0, scA); scales(w1, scB);
    const uint8_t * y = C.b + 256 * task + 4 * t;
    int acc[4] = { 0, 0, 0, 0 };
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const uint32_t hmA = lds4<R>(w0 + 16 * half + 4 * t), hmB = lds4<R>(w1 + 16 * half + 4 * t);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t qa = lds4<R>(w0 + 32 + 32 * h + 16 * half + 4 * t), qb = lds4<R>(w1 + 32 + 32 * h + 16 * half + 4 * t);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                const int g = 8 * h + 2 * jj + half, bit = 4 * h + jj;   // compile time
                const uint32_t a0 = ((qa >> (2 * jj)) & 0x03030303u) | (((hmA >> bit) & 0x01010101u) << 2);
                const uint32_t a1 = ((qb >> (2 * jj)) & 0x03030303u) | (((hmB >> bit) & 0x01010101u) << 2);
                const uint32_t b0 = *(const uint32_t *)(y + 16 * g);
                int c[4];
                mma_s8_16x8x16(c, a0, a1, b0);
                const int sa = (g & 3) == 0 ? sbyte<0>(scA[g >> 2]) : (g & 3) == 1 ? sbyte<1>(scA[g >> 2]) : (g & 3) == 2 ? sbyte<2>(scA[g >> 2]) : sbyte<3>(scA[g >> 2]);
                const int sb = (g & 3) == 0 ? sbyte<0>(scB[g >> 2]) : (g & 3) == 1 ? sbyte<1>(scB[g >> 2]) : (g & 3) == 2 ? sbyte<2>(scB[g >> 2]) : sbyte<3>(scB[g >> 2]);
                acc[0] += sa * c[0]; acc[1] += sa * c[1]; acc[2] += sb * c[2]; acc[3] += sb * c[3];
            }
        }
    }
    auto offs = [](const int4 & sa, const int4 & sb, const uint32_t (&sc)[4]) {
        int o = dp2a_lo_ss(sa.x, sc[0], 0);
        o = dp2a_hi_ss(sa.y, sc[0], o); o = dp2a_lo_ss(sa.z, sc[1], o); o = dp2a_hi_ss(sa.w, sc[1], o);
        o = dp2a_lo_ss(sb.x, sc[2], o); o = dp2a_hi_ss(sb.y, sc[2], o); o = dp2a_lo_ss(sb.z, sc[3], o);
        return dp2a_hi_ss(sb.w, sc[3], o);
    };
    const int4 s0a = lds128(C.c0 + A.off_s16 + 32 * task), s0b = lds128(C.c0 + A.off_s16 + 32 * task + 16);
    const int4 s1a = lds128(C.c1 + A.off_s16 + 32 * task), s1b = lds128(C.c1 + A.off_s16 + 32 * task + 16);
    const float yd0 = *(const float *)(C.c0 + A.off_d + 4 * task), yd1 = *(const float *)(C.c1 + A.off_d + 4 * task);
    const float dA = h2f(lds_u16(w0 + 108)), dB = h2f(lds_u16(w1 + 108));
    facc[0] += (dA * yd0) * (float)(acc[0] - 4 * offs(s0a, s0b, scA));
    facc[1] += (dA * yd1) * (float)(acc[1] - 4 * offs(s1a, s1b, scA));
    facc[2] += (dB * yd0) * (float)(acc[2] - 4 * offs(s0a, s0b, scB));
    facc[3] += (dB * yd1) * (float)(acc[3] - 4 * offs(s1a, s1b, scB));
}
template <> __device__ __forceinline__ void mma_task<T_Q3_K>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) {
    if (((uintptr_t)w0 & 2) != 0) mma_q3_task<2>(w0, w1, C, A, task, t, facc);
    else                          mma_q3_task<0>(w0, w1, C, A, task, t, facc);
}

// Q6_K: 210-byte superblocks (ql[128] | qh[64] | int8 scales[16] | d), sixteen 16-weight scale groups -> sixteen m16n8k16 products per task.
// Group (half n, quarter q, sixteen is) = weights 128 n + 32 q + 16 is .. + 15: low nibbles (q < 2) or high nibbles (q >= 2) of
// ql[64 n + 32 (q & 1) + 16 is ..], bits 2q, 2q+1 of qh[32 n + 16 is ..], scale index 8 n + 2 q + is = (first weight) / 16.  The "- 32" of
// the codes is sum_ch scale_ch * (16-sum of the activations)_ch.  Superblocks are only 2-byte aligned: R = 2 for odd tasks of a row slice.
template <int R>
__device__ __forceinline__ void mma_q6_task(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) {
    uint32_t scA[4], scB[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { scA[i] = lds4<R>(w0 + 192 + 4 * i); scB[i] = lds4<R>(w1 + 192 + 4 * i); }
    const uint8_t * y = C.b + 256 * task + 4 * t;
    int acc[4] = { 0, 0, 0, 0 };
#pragma unroll
    for (int n = 0; n < 2; ++n) {
#pragma unroll
        for (int is = 0; is < 2; ++is) {
            const int o = 16 * is + 4 * t;
            const uint32_t la0 = lds4<R>(w0 + 64 * n + o), lb0 = lds4<R>(w0 + 64 * n + 32 + o), h0 = lds4<R>(w0 + 128 + 32 * n + o);
            const uint32_t la1 = lds4<R>(w1 + 64 * n + o), lb1 = lds4<R>(w1 + 64 * n + 32 + o), h1 = lds4<R>(w1 + 128 + 32 * n + o);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const uint32_t l0 = (q & 1) ? lb0 : la0, l1 = (q & 1) ? lb1 : la1;
                const uint32_t a0 = ((q < 2 ? l0 : l0 >> 4) & 0x0F0F0F0Fu) | ((q == 0 ? h0 << 4 : q == 1 ? h0 << 2 : q == 2 ? h0 : h0 >> 2) & 0x30303030u);
                const uint32_t a1 = ((q < 2 ? l1 : l1 >> 4) & 0x0F0F0F0Fu) | ((q == 0 ? h1 << 4 : q == 1 ? h1 << 2 : q == 2 ? h1 : h1 >> 2) & 0x30303030u);
                const uint32_t b0 = *(const uint32_t *)(y + 128 * n + 32 * q + 16 * is);
                int c[4];
                mma_s8_16x8x16(c, a0, a1, b0);
                const int ch = 8 * n + 2 * q + is;                      // scale index (compile time)
                const int sa = (ch & 3) == 0 ? sbyte<0>(scA[ch >> 2]) : (ch & 3) == 1 ? sbyte<1>(scA[ch >> 2]) : (ch & 3) == 2 ? sbyte<2>(scA[ch >> 2]) : sbyte<3>(scA[ch >> 2]);
                const int sb = (ch & 3) == 0 ? sbyte<0>(scB[ch >> 2]) : (ch & 3) == 1 ? sbyte<1>(scB[ch >> 2]) : (ch & 3) == 2 ? sbyte<2>(scB[ch >> 2]) : sbyte<3>(scB[ch >> 2]);
                acc[0] += sa * c[0]; acc[1] += sa * c[1]; acc[2] += sb * c[2]; acc[3] += sb * c[3];
            }
        }
    }
    // offsets: sum over the sixteen groups of scale x (16-sum of the column's activations), two groups per dp2a
    auto offs = [](const int4 & sa, const int4 & sb, const uint32_t (&sc)[4]) {
        int o = dp2a_lo_ss(sa.x, sc[0], 0);
        o = dp2a_hi_ss(sa.y, sc[0], o); o = dp2a_lo_ss(sa.z, sc[1], o); o = dp2a_hi_ss(sa.w, sc[1], o);
        o = dp2a_lo_ss(sb.x, sc[2], o); o = dp2a_hi_ss(sb.y, sc[2], o); o = dp2a_lo_ss(sb.z, sc[3], o);
        return dp2a_hi_ss(sb.w, sc[3], o);
    };
    const int4 s0a = lds128(C.c0 + A.off_s16 + 32 * task), s0b = lds128(C.c0 + A.off_s16 + 32 * task + 16);
    const int4 s1a = lds128(C.c1 + A.off_s16 + 32 * task), s1b = lds128(C.c1 + A.off_s16 + 32 * task + 16);
    const float yd0 = *(const float *)(C.c0 + A.off_d + 4 * task), yd1 = *(const float *)(C.c1 + A.off_d + 4 * task);
    const float dA = h2f(lds_u16(w0 + 208)), dB = h2f(lds_u16(w1 + 208));
    facc[0] += (dA * yd0) * (float)(acc[0] - 32 * offs(s0a, s0b, scA));
    facc[1] += (dA * yd1) * (float)(acc[1] - 32 * offs(s1a, s1b, scA));
    facc[2] += (dB * yd0) * (float)(acc[2] - 32 * offs(s0a, s0b, scB));
    facc[3] += (dB * yd1) * (float)(acc[3] - 32 * offs(s1a, s1b, scB));
}
template <> __device__ __forceinline__ void mma_task<T_Q6_K>(const uint8_t * w0, const uint8_t * w1, const mma_cols & C, const mma_act & A, int task, int t, float (&facc)[4]) {
    // (w0 and w1 are a multiple of the 16-byte aligned row pitch apart: same residue)
    if (((uintptr_t)w0 & 2) != 0) mma_q6_task<2>(w0, w1, C, A, task, t, facc);
    else                          mma_q6_task<0>(w0, w1, C, A, task, t, facc);
}

} // namespace b200
