// b200_sb_tasks.cuh — per-lane "task" dot products of the superblock mat-vec kernel (mmvq_sb.cu): a task = 256 (Q8_0: 128)
// consecutive weights of one row against the per-task activation record.  Pure per-thread code, split from the kernel file so
// that tests/hostemu can compile it for the host (B200_HOST_EMU: the few inline-PTX helpers get C++ restatements of the PTX
// semantics) and check the decode logic against the oracle in the CPU-only suite.
#pragma once
#include "b200_quants.cuh"

namespace b200 {

// mixed-sign dp4a: bytes of a are unsigned, bytes of b signed
#ifndef B200_HOST_EMU
__device__ __forceinline__ int dp4a_us(uint32_t a, int b, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
#else
inline int dp4a_us(uint32_t a, int b, int c) { for (int i = 0; i < 4; ++i) c += (int)((a >> (8 * i)) & 0xFF) * (int)(int8_t)(b >> (8 * i)); return c; }
#endif

// ----------------------------------------------------------------------------- task geometry
// TASK_W weights per task, TASK_B bytes; LPR lanes per row.
template <int T> struct sbfmt;
template <> struct sbfmt<T_Q4_K> { static constexpr int TASK_W = 256, TASK_B = 144, LPR = 16, KQ = 1; };
template <> struct sbfmt<T_Q5_K> { static constexpr int TASK_W = 256, TASK_B = 176, LPR = 16, KQ = 1; };
template <> struct sbfmt<T_Q6_K> { static constexpr int TASK_W = 256, TASK_B = 210, LPR = 16, KQ = 1; };
template <> struct sbfmt<T_Q4_0> { static constexpr int TASK_W = 256, TASK_B = 144, LPR = 16, KQ = 0; };
template <> struct sbfmt<T_Q8_0> { static constexpr int TASK_W = 128, TASK_B = 136, LPR = 32, KQ = 0; };
// SURVEY §8f-2 formats: task dot products written and host-verified (tests/hostemu), dispatched by mmvq_sb.cu
// like the hot-path formats (GPU check: tests/test_gpu_next_formats.py)
template <> struct sbfmt<T_Q5_0> { static constexpr int TASK_W = 256, TASK_B = 176, LPR = 16, KQ = 0; };
template <> struct sbfmt<T_IQ4_NL> { static constexpr int TASK_W = 256, TASK_B = 144, LPR = 16, KQ = 0; };
template <> struct sbfmt<T_IQ4_XS> { static constexpr int TASK_W = 256, TASK_B = 136, LPR = 16, KQ = 1; };
template <> struct sbfmt<T_Q4_1> { static constexpr int TASK_W = 256, TASK_B = 160, LPR = 16, KQ = 0; };   // needs the Q8_1 s values: see task_dot<T_Q4_1>
template <> struct sbfmt<T_Q5_1> { static constexpr int TASK_W = 256, TASK_B = 192, LPR = 16, KQ = 0; };
template <> struct sbfmt<T_Q2_K> { static constexpr int TASK_W = 256, TASK_B = 84,  LPR = 16, KQ = 1; };
template <> struct sbfmt<T_Q3_K> { static constexpr int TASK_W = 256, TASK_B = 110, LPR = 16, KQ = 1; };

// Activation record in shared memory: one SB_REC-byte record per act-task (256 consecutive activations), task t at rec + t * SB_REC:
//   +0   q    : 256 int8 (chunk j = values 16 j .. 16 j + 15 at +16 j)
//   +256 s32  : eight int32 sums of 32 values
//   +288 s16  : sixteen int16 sums of 16 values
//   +320 h32  : the eight 32-sums again as int16 (operand of dp2a against packed 6-bit mins)
//   +336 d    : Q8_K family: one float;  Q8_0 family: eight floats (fp16-rounded block scales)
// SB_REC = 23 x 16: an odd number of 16-byte units, so lanes working on consecutive tasks hit different bank groups with every
// LDS.128 (conflict-free), and every load address is "task base + immediate" -- no address arithmetic inside the dot products.
constexpr int SB_REC = 368, SB_OFF_S32 = 256, SB_OFF_S16 = 288, SB_OFF_H32 = 320, SB_OFF_D = 336;
struct sb_act {
    int32_t ntask, bytes;
};
__host__ __device__ inline sb_act make_sb_act(int64_t K) {
    sb_act A;
    A.ntask = (int32_t)(K / 256);
    A.bytes = A.ntask * SB_REC;
    return A;
}

// ----------------------------------------------------------------------------- in-kernel activation quantizer
// Half a warp (16 lanes) quantizes act-task t: lane l owns values 16 l .. 16 l + 15 (= chunk l of the record), so the chunk, its
// 16-sum and most of the amax search are lane-local; 4 shuffle rounds, and two tasks per warp run side by side.
// Shuffles use xor distances < 16, i.e. they never cross the half-warp; all 32 lanes must call this together.
// Numerics: exactly ggml-cpu's quantize_row_q8_K (KQ) / AVX2 quantize_row_q8_0 (see b200_quants.cuh).
// Q81S (Q8_0 family only): the H32 slot receives block_q8_1.s = fp16(d_unrounded * sum of the block's codes) instead of the int16 sums
// (weight formats with a minimum, Q4_1 / Q5_1).  Q81S = false is the code path of the hot-path formats, unchanged.
// The arithmetic is sb_quantize_core (shared with the planar records of the mma path, b200_sb_mma.cuh); the wrappers only differ in
// where the results are stored.
struct sb_qtask {
    int4  pk;        // this lane's 16 codes, packed
    int   s, s2;     // sum of the lane's 16 codes; sum of the 32-value block (lanes 2b, 2b+1)
    float d;         // KQ: the task's scale 1 / iscale (0 for an all-zero task); else the block's fp16-rounded scale
    float dun;       // Q8_0 family: the block's unrounded scale amax / 127
};
template <bool KQ> __device__ __forceinline__ sb_qtask sb_quantize_core(const float * __restrict__ x, bool valid, int t) {
    const int l = threadIdx.x & 15;
    float v[16];
    if (valid) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float4 f = load_f4(x + (size_t)t * 256 + 16 * l + 4 * i); v[4 * i] = f.x; v[4 * i + 1] = f.y; v[4 * i + 2] = f.z; v[4 * i + 3] = f.w; }
    } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = 0.0f;
    }
    sb_qtask r;
    int q[16];
    r.dun = 0.0f; r.d = 0.0f;
    if constexpr (KQ) {
        float amax = 0.0f, vmax = 0.0f; int imax = 0;
#pragma unroll
        for (int i = 0; i < 16; ++i) { const float ax = fabsf(v[i]); if (ax > amax) { amax = ax; vmax = v[i]; imax = 16 * l + i; } }
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) {
            const float oa = __shfl_xor_sync(0xffffffffu, amax, o), ov = __shfl_xor_sync(0xffffffffu, vmax, o);
            const int   oi = __shfl_xor_sync(0xffffffffu, imax, o);
            if (oa > amax || (oa == amax && oi < imax)) { amax = oa; vmax = ov; imax = oi; }
        }
        if (amax != 0.0f) {
            const float iscale = __fdiv_rn(-127.0f, vmax);
#pragma unroll
            for (int i = 0; i < 16; ++i) q[i] = min(127, __float2int_rn(iscale * v[i]));
            r.d = __fdiv_rn(1.0f, iscale);
        } else {
#pragma unroll
            for (int i = 0; i < 16; ++i) q[i] = 0;
        }
    } else {
        float amax = 0.0f;
#pragma unroll
        for (int i = 0; i < 16; ++i) amax = fmaxf(amax, fabsf(v[i]));
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));               // 32-value block = lanes 2b, 2b+1
        const float id = amax != 0.0f ? __fdiv_rn(127.0f, amax) : 0.0f;
#pragma unroll
        for (int i = 0; i < 16; ++i) q[i] = __float2int_rn(v[i] * id);
        r.dun = __fdiv_rn(amax, 127.0f);
        r.d = __half2float(__float2half_rn(r.dun));
    }
    int s = 0;
    int * pw = &r.pk.x;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        pw[w] = (int)((uint32_t)(q[4 * w] & 0xFF) | ((uint32_t)(q[4 * w + 1] & 0xFF) << 8) | ((uint32_t)(q[4 * w + 2] & 0xFF) << 16) | ((uint32_t)(q[4 * w + 3] & 0xFF) << 24));
        s += q[4 * w] + q[4 * w + 1] + q[4 * w + 2] + q[4 * w + 3];
    }
    r.s = s;
    r.s2 = s + __shfl_xor_sync(0xffffffffu, s, 1);
    return r;
}

template <bool KQ, bool Q81S = false> __device__ __forceinline__ void sb_quantize_task_h(const float * __restrict__ x, bool valid, uint8_t * rec, int t) {
    const int l = threadIdx.x & 15;
    const sb_qtask r = sb_quantize_core<KQ>(x, valid, t);
    uint8_t * rb = rec + (size_t)t * SB_REC;
    if (valid) {
        if constexpr (KQ) { if (l == 0) *(float *)(rb + SB_OFF_D) = r.d; }
        else              { if ((l & 1) == 0) *(float *)(rb + SB_OFF_D + 4 * (l >> 1)) = r.d; }
        *(int4 *)(rb + 16 * l) = r.pk;
        *(int16_t *)(rb + SB_OFF_S16 + 2 * l) = (int16_t)r.s;
        if ((l & 1) == 0) {
            *(int32_t *)(rb + SB_OFF_S32 + 4 * (l >> 1)) = r.s2;
            if constexpr (!KQ && Q81S) *(__half *)(rb + SB_OFF_H32 + 2 * (l >> 1)) = __float2half_rn(__fmul_rn(r.dun, (float)r.s2));
            else                       *(int16_t *)(rb + SB_OFF_H32 + 2 * (l >> 1)) = (int16_t)r.s2;   // |s2| <= 32 * 127
        }
    }
}

__device__ __forceinline__ int4 lds128(const uint8_t * p) { return *(const int4 *)p; }
// d = c + a.lo16 * b.byte0 + a.hi16 * b.byte1 (lo) / b.byte2, b.byte3 (hi); a halves signed, b bytes unsigned (su) or signed (ss)
#ifndef B200_HOST_EMU
__device__ __forceinline__ int dp2a_lo_su(int a, uint32_t b, int c) { int d; asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_hi_su(int a, uint32_t b, int c) { int d; asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_lo_ss(int a, uint32_t b, int c) { int d; asm("dp2a.lo.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_hi_ss(int a, uint32_t b, int c) { int d; asm("dp2a.hi.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
template <int B> __device__ __forceinline__ int ubyte(uint32_t x) { return (int)__byte_perm(x, 0, 0x4440 + B); }             // zero-extended byte B
// sign-extended byte B: PTX prmt in default mode replicates the sign of the selected byte when bit 3 of a selector nibble is set
// (__byte_perm only honours 3 selector bits, hence the inline PTX)
template <int B> __device__ __forceinline__ int sbyte(uint32_t x) {
    int d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(x), "r"(0u), "r"((uint32_t)(B | ((8 | B) << 4) | ((8 | B) << 8) | ((8 | B) << 12))));
    return d;
}
#else   // host restatements of the PTX semantics above (tests/hostemu)
inline int dp2a_emu(int a, uint32_t b, int c, int first_byte, bool b_signed) {
    const int lo = (int)(int16_t)(a & 0xFFFF), hi = (int)(int16_t)((uint32_t)a >> 16);
    const uint32_t b0 = (b >> (8 * first_byte)) & 0xFF, b1 = (b >> (8 * first_byte + 8)) & 0xFF;
    return c + lo * (b_signed ? (int)(int8_t)b0 : (int)b0) + hi * (b_signed ? (int)(int8_t)b1 : (int)b1);
}
inline int dp2a_lo_su(int a, uint32_t b, int c) { return dp2a_emu(a, b, c, 0, false); }
inline int dp2a_hi_su(int a, uint32_t b, int c) { return dp2a_emu(a, b, c, 2, false); }
inline int dp2a_lo_ss(int a, uint32_t b, int c) { return dp2a_emu(a, b, c, 0, true); }
inline int dp2a_hi_ss(int a, uint32_t b, int c) { return dp2a_emu(a, b, c, 2, true); }
template <int B> inline int ubyte(uint32_t x) { return (int)((x >> (8 * B)) & 0xFF); }
template <int B> inline int sbyte(uint32_t x) { return (int)(int8_t)((x >> (8 * B)) & 0xFF); }
#endif

// ----------------------------------------------------------------------------- task dot products
// `w` points at the task's first byte in the shared-memory stage, `rec` at the activation record, `t` = task index in the row.
template <int T> __device__ __forceinline__ float task_dot(const uint8_t * w, const uint8_t * rec, int t);

// one 64-weight chunk C of a Q4_K / Q5_K superblock: sub-block 2C in the low nibbles (scale sc0), 2C+1 in the high ones (sc1)
template <int C, bool FIVE>
__device__ __forceinline__ void q45_chunk(const uint8_t * qs, const uint32_t (&qh)[8], const uint8_t * a, int sc0, int sc1, int & acc_s) {
    const int4 qa = lds128(qs + 32 * C), qb = lds128(qs + 32 * C + 16);
    const uint32_t q[8] = { (uint32_t)qa.x, (uint32_t)qa.y, (uint32_t)qa.z, (uint32_t)qa.w, (uint32_t)qb.x, (uint32_t)qb.y, (uint32_t)qb.z, (uint32_t)qb.w };
    int p0 = 0, p1 = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int4 ylo = lds128(a + (4 * C + h) * 16);                              // values 64C + 16h ..   (sub-block 2C)
        const int4 yhi = lds128(a + (4 * C + 2 + h) * 16);                          // values 64C + 32 + 16h (sub-block 2C+1)
        const int yl[4] = { ylo.x, ylo.y, ylo.z, ylo.w }, yh[4] = { yhi.x, yhi.y, yhi.z, yhi.w };
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t qq = q[4 * h + i];
            if constexpr (FIVE) {
                const uint32_t hb = qh[4 * h + i] >> (2 * C);
                p0 = __dp4a((int)((qq & 0x0F0F0F0F) | ((hb & 0x01010101) << 4)), yl[i], p0);
                p1 = __dp4a((int)(((qq >> 4) & 0x0F0F0F0F) | ((hb & 0x02020202) << 3)), yh[i], p1);
            } else {
                p0 = __dp4a((int)(qq & 0x0F0F0F0F), yl[i], p0);
                p1 = dp4a_us(qq & 0xF0F0F0F0u, yh[i], p1);                          // 16 x (high nibbles . y)
            }
        }
    }
    if constexpr (!FIVE) p1 >>= 4;                                                  // exact: a multiple of 16
    acc_s += sc0 * p0 + sc1 * p1;
}

template <bool FIVE> __device__ __forceinline__ float q45_task(const uint8_t * w, const uint8_t * rec, int t) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
    const int4 hdr = lds128(w);                                     // d | dmin | scales[12]
    const int4 h32 = lds128(a + SB_OFF_H32);                        // eight 32-sums, int16
    uint32_t qh[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    if constexpr (FIVE) {
        const int4 ha = lds128(w + 16), hb = lds128(w + 32);
        qh[0] = ha.x; qh[1] = ha.y; qh[2] = ha.z; qh[3] = ha.w; qh[4] = hb.x; qh[5] = hb.y; qh[6] = hb.z; qh[7] = hb.w;
    }
    const uint8_t * qs = w + (FIVE ? 48 : 16);
    // the 6-bit (scale, min) pairs of get_scale_min_k4, four sub-blocks per word
    const uint32_t s0 = hdr.y, s1 = hdr.z, s2 = hdr.w;
    const uint32_t sc_lo = s0 & 0x3F3F3F3Fu, mn_lo = s1 & 0x3F3F3F3Fu;                                   // sub-blocks 0..3
    const uint32_t sc_hi = (s2 & 0x0F0F0F0Fu) | ((s0 >> 2) & 0x30303030u);                               // sub-blocks 4..7
    const uint32_t mn_hi = ((s2 >> 4) & 0x0F0F0F0Fu) | ((s1 >> 2) & 0x30303030u);
    int acc_m = dp2a_lo_su(h32.x, mn_lo, 0);                        // sum_j min_j * (sum of the 32 activations of sub-block j)
    acc_m = dp2a_hi_su(h32.y, mn_lo, acc_m);
    acc_m = dp2a_lo_su(h32.z, mn_hi, acc_m);
    acc_m = dp2a_hi_su(h32.w, mn_hi, acc_m);
    int acc_s = 0;
    q45_chunk<0, FIVE>(qs, qh, a, ubyte<0>(sc_lo), ubyte<1>(sc_lo), acc_s);
    q45_chunk<1, FIVE>(qs, qh, a, ubyte<2>(sc_lo), ubyte<3>(sc_lo), acc_s);
    q45_chunk<2, FIVE>(qs, qh, a, ubyte<0>(sc_hi), ubyte<1>(sc_hi), acc_s);
    q45_chunk<3, FIVE>(qs, qh, a, ubyte<2>(sc_hi), ubyte<3>(sc_hi), acc_s);
    const float yd = *(const float *)(a + SB_OFF_D);
    const float d = h2f((uint32_t)hdr.x & 0xFFFF) * yd, dmin = h2f((uint32_t)hdr.x >> 16) * yd;
    return d * (float)acc_s - dmin * (float)acc_m;
}
template <> __device__ __forceinline__ float task_dot<T_Q4_K>(const uint8_t * w, const uint8_t * rec, int t) { return q45_task<false>(w, rec, t); }
template <> __device__ __forceinline__ float task_dot<T_Q5_K>(const uint8_t * w, const uint8_t * rec, int t) { return q45_task<true>(w, rec, t); }

// Q4_0: task = 8 blocks of 18 bytes = 144 bytes (16-byte aligned), act-task == task
template <> __device__ __forceinline__ float task_dot<T_Q4_0>(const uint8_t * w, const uint8_t * rec, int t) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
    uint32_t ww[37];
#pragma unroll
    for (int i = 0; i < 9; ++i) { const int4 v = lds128(w + 16 * i); ww[4 * i] = v.x; ww[4 * i + 1] = v.y; ww[4 * i + 2] = v.z; ww[4 * i + 3] = v.w; }
    ww[36] = 0;
    const int4 sa = lds128(a + SB_OFF_S32), sb = lds128(a + SB_OFF_S32 + 16);
    const int s32[8] = { sa.x, sa.y, sa.z, sa.w, sb.x, sb.y, sb.z, sb.w };
    const int4 da = lds128(a + SB_OFF_D), db = lds128(a + SB_OFF_D + 16);
    const float yd[8] = { __int_as_float(da.x), __int_as_float(da.y), __int_as_float(da.z), __int_as_float(da.w),
                          __int_as_float(db.x), __int_as_float(db.y), __int_as_float(db.z), __int_as_float(db.w) };
    float acc = 0.0f;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
        // block b starts at byte 18 b = word 4.5 b: even b word-aligned, odd b half-word shifted (all compile-time)
        const int w0 = (18 * b) / 4;
        const bool odd = (b & 1) != 0;
        uint32_t q[4];
        uint32_t dbits;
        if (!odd) {
            dbits = ww[w0] & 0xFFFF;
#pragma unroll
            for (int i = 0; i < 4; ++i) q[i] = __funnelshift_r(ww[w0 + i], ww[w0 + i + 1], 16);
        } else {
            dbits = ww[w0] >> 16;
#pragma unroll
            for (int i = 0; i < 4; ++i) q[i] = ww[w0 + 1 + i];
        }
        const int4 ylo = lds128(a + (2 * b) * 16), yhi = lds128(a + (2 * b + 1) * 16);
        const int yl[4] = { ylo.x, ylo.y, ylo.z, ylo.w }, yh[4] = { yhi.x, yhi.y, yhi.z, yhi.w };
        int p0 = 0, p1 = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            p0 = __dp4a((int)(q[i] & 0x0F0F0F0F), yl[i], p0);
            p1 = dp4a_us(q[i] & 0xF0F0F0F0u, yh[i], p1);
        }
        const int s = p0 + (p1 >> 4) - 8 * s32[b];
        acc += (float)s * h2f(dbits) * yd[b];
    }
    return acc;
}

// Q8_0: task = 4 blocks of 34 bytes = 136 bytes (8-byte aligned); two tasks per 256-value act-task
template <> __device__ __forceinline__ float task_dot<T_Q8_0>(const uint8_t * w, const uint8_t * rec, int t) {
    uint32_t ww[35];
#pragma unroll
    for (int i = 0; i < 17; ++i) { const uint2 v = *(const uint2 *)(w + 8 * i); ww[2 * i] = v.x; ww[2 * i + 1] = v.y; }
    ww[34] = 0;
    const int at = t >> 1, hf = t & 1;                                             // act-task, which half of it
    const uint8_t * a = rec + (size_t)at * SB_REC + hf * 128;                      // q chunks 8 hf .. 8 hf + 7
    const int4 dv = lds128(rec + (size_t)at * SB_REC + SB_OFF_D + hf * 16);
    const float yd[4] = { __int_as_float(dv.x), __int_as_float(dv.y), __int_as_float(dv.z), __int_as_float(dv.w) };
    float acc = 0.0f;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
        const int w0 = (34 * b) / 4;
        const bool odd = (b & 1) != 0;                                             // 34 b mod 4 = 2 for odd b
        const uint32_t dbits = odd ? (ww[w0] >> 16) : (ww[w0] & 0xFFFF);
        const int4 y0 = lds128(a + (2 * b) * 16), y1 = lds128(a + (2 * b + 1) * 16);
        const int y[8] = { y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w };
        int s = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const uint32_t q = odd ? ww[w0 + 1 + i] : __funnelshift_r(ww[w0 + i], ww[w0 + i + 1], 16);
            s = __dp4a((int)q, y[i], s);
        }
        acc += (float)s * (h2f(dbits) * yd[b]);
    }
    return acc;
}

// Q6_K: 210-byte superblocks are only 2-byte aligned: aligned words + one run-time funnel shift (0 or 16 bits)
template <> __device__ __forceinline__ float task_dot<T_Q6_K>(const uint8_t * w, const uint8_t * rec, int t) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
    const uint32_t sh = ((uint32_t)(uintptr_t)w & 2) * 8;
    const uint32_t * wa = (const uint32_t *)((uintptr_t)w & ~(uintptr_t)3);
    auto word = [&](int i) { return __funnelshift_r(wa[i], wa[i + 1], sh); };     // 32-bit word i of the superblock
    const int4 sa = lds128(a + SB_OFF_S16), sb = lds128(a + SB_OFF_S16 + 16);
    const int s16w[8] = { sa.x, sa.y, sa.z, sa.w, sb.x, sb.y, sb.z, sb.w };       // sixteen 16-sums, int16 pairs
    int tot = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint32_t scw0 = word(48 + 2 * h), scw1 = word(48 + 2 * h + 1);       // int8 scales[8h .. 8h+7]
        // value = d * sc * (q - 32): the "- 32" part is sum_g sc_g * (16-sum)_g, two groups per dp2a
        int off = dp2a_lo_ss(s16w[4 * h], scw0, 0);
        off = dp2a_hi_ss(s16w[4 * h + 1], scw0, off);
        off = dp2a_lo_ss(s16w[4 * h + 2], scw1, off);
        off = dp2a_hi_ss(s16w[4 * h + 3], scw1, off);
        tot -= 32 * off;
#pragma unroll
        for (int j = 0; j < 2; ++j) {                                              // l-range 16 j .. 16 j + 15
            int p[4] = { 0, 0, 0, 0 };
            const int4 yv0 = lds128(a + (8 * h + j) * 16), yv1 = lds128(a + (8 * h + j + 2) * 16);
            const int4 yv2 = lds128(a + (8 * h + j + 4) * 16), yv3 = lds128(a + (8 * h + j + 6) * 16);
            const int ya[4] = { yv0.x, yv0.y, yv0.z, yv0.w }, yb[4] = { yv1.x, yv1.y, yv1.z, yv1.w };
            const int yc[4] = { yv2.x, yv2.y, yv2.z, yv2.w }, yd4[4] = { yv3.x, yv3.y, yv3.z, yv3.w };
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint32_t la = word(16 * h + 4 * j + i), lb = word(16 * h + 8 + 4 * j + i), qh = word(32 + 8 * h + 4 * j + i);
                p[0] = __dp4a((int)((la & 0x0F0F0F0F)        | ((qh << 4) & 0x30303030)), ya[i], p[0]);
                p[1] = __dp4a((int)((lb & 0x0F0F0F0F)        | ((qh << 2) & 0x30303030)), yb[i], p[1]);
                p[2] = __dp4a((int)(((la >> 4) & 0x0F0F0F0F) | ( qh       & 0x30303030)), yc[i], p[2]);
                p[3] = __dp4a((int)(((lb >> 4) & 0x0F0F0F0F) | ((qh >> 2) & 0x30303030)), yd4[i], p[3]);
            }
            // scales[8h + j + 2g] multiplies p[g]
            if (j == 0) tot += sbyte<0>(scw0) * p[0] + sbyte<2>(scw0) * p[1] + sbyte<0>(scw1) * p[2] + sbyte<2>(scw1) * p[3];
            else        tot += sbyte<1>(scw0) * p[0] + sbyte<3>(scw0) * p[1] + sbyte<1>(scw1) * p[2] + sbyte<3>(scw1) * p[3];
        }
    }
    const float d = h2f(word(52) & 0xFFFF) * *(const float *)(a + SB_OFF_D);
    return d * (float)tot;
}

// ---- SURVEY §8f-2 formats (host-verified; see sbfmt above) --------------------------------------------------------------
// Q5_0: task = 8 blocks of 22 bytes = 176 bytes (16-byte aligned); block = d (2 B), 32 fifth bits (4 B), 16 nibble bytes
template <> __device__ __forceinline__ float task_dot<T_Q5_0>(const uint8_t * w, const uint8_t * rec, int t) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
    uint32_t ww[45];
#pragma unroll
    for (int i = 0; i < 11; ++i) { const int4 v = lds128(w + 16 * i); ww[4 * i] = v.x; ww[4 * i + 1] = v.y; ww[4 * i + 2] = v.z; ww[4 * i + 3] = v.w; }
    ww[44] = 0;
    const int4 sa = lds128(a + SB_OFF_S32), sb = lds128(a + SB_OFF_S32 + 16);
    const int s32[8] = { sa.x, sa.y, sa.z, sa.w, sb.x, sb.y, sb.z, sb.w };
    const int4 da = lds128(a + SB_OFF_D), db = lds128(a + SB_OFF_D + 16);
    const float yd[8] = { __int_as_float(da.x), __int_as_float(da.y), __int_as_float(da.z), __int_as_float(da.w),
                          __int_as_float(db.x), __int_as_float(db.y), __int_as_float(db.z), __int_as_float(db.w) };
    float acc = 0.0f;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
        // block b starts at byte 22 b = word 5.5 b: even b word-aligned, odd b half-word shifted (all compile-time)
        const int w0 = (22 * b) / 4;
        const bool odd = (b & 1) != 0;
        uint32_t q[4], dbits, qh;
        if (!odd) {
            dbits = ww[w0] & 0xFFFF;
            qh = __funnelshift_r(ww[w0], ww[w0 + 1], 16);
#pragma unroll
            for (int i = 0; i < 4; ++i) q[i] = __funnelshift_r(ww[w0 + 1 + i], ww[w0 + 2 + i], 16);
        } else {
            dbits = ww[w0] >> 16;
            qh = ww[w0 + 1];
#pragma unroll
            for (int i = 0; i < 4; ++i) q[i] = ww[w0 + 2 + i];
        }
        const int4 ylo = lds128(a + (2 * b) * 16), yhi = lds128(a + (2 * b + 1) * 16);
        const int y[8] = { ylo.x, ylo.y, ylo.z, ylo.w, yhi.x, yhi.y, yhi.z, yhi.w };
        const int s = q5_block_dot(q, qh, y) - 16 * s32[b];
        acc += (h2f(dbits) * yd[b]) * (float)s;
    }
    return acc;
}

// IQ4_NL: the Q4_0 task (8 blocks of 18 bytes) with the nibbles mapped through the non-linear codebook (two byte permutes per word)
template <> __device__ __forceinline__ float task_dot<T_IQ4_NL>(const uint8_t * w, const uint8_t * rec, int t) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
    uint32_t ww[37];
#pragma unroll
    for (int i = 0; i < 9; ++i) { const int4 v = lds128(w + 16 * i); ww[4 * i] = v.x; ww[4 * i + 1] = v.y; ww[4 * i + 2] = v.z; ww[4 * i + 3] = v.w; }
    ww[36] = 0;
    const int4 da = lds128(a + SB_OFF_D), db = lds128(a + SB_OFF_D + 16);
    const float yd[8] = { __int_as_float(da.x), __int_as_float(da.y), __int_as_float(da.z), __int_as_float(da.w),
                          __int_as_float(db.x), __int_as_float(db.y), __int_as_float(db.z), __int_as_float(db.w) };
    float acc = 0.0f;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
        const int w0 = (18 * b) / 4;
        const bool odd = (b & 1) != 0;
        uint32_t q[4], dbits;
        if (!odd) {
            dbits = ww[w0] & 0xFFFF;
#pragma unroll
            for (int i = 0; i < 4; ++i) q[i] = __funnelshift_r(ww[w0 + i], ww[w0 + i + 1], 16);
        } else {
            dbits = ww[w0] >> 16;
#pragma unroll
            for (int i = 0; i < 4; ++i) q[i] = ww[w0 + 1 + i];
        }
        const int4 ylo = lds128(a + (2 * b) * 16), yhi = lds128(a + (2 * b + 1) * 16);
        const int yl[4] = { ylo.x, ylo.y, ylo.z, ylo.w }, yh[4] = { yhi.x, yhi.y, yhi.z, yhi.w };
        int s = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            s = __dp4a((int)iq4nl_lookup4(q[i]), yl[i], s);
            s = __dp4a((int)iq4nl_lookup4(q[i] >> 4), yh[i], s);
        }
        acc += (yd[b] * h2f(dbits)) * (float)s;
    }
    return acc;
}

// IQ4_XS: 136-byte superblocks are 8-byte aligned: 64-bit loads.  words: d | scales_h, scales_l, then 32 words of qs
template <> __device__ __forceinline__ float task_dot<T_IQ4_XS>(const uint8_t * w, const uint8_t * rec, int t) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
    uint32_t ww[34];
#pragma unroll
    for (int i = 0; i < 17; ++i) { const uint2 v = *(const uint2 *)(w + 8 * i); ww[2 * i] = v.x; ww[2 * i + 1] = v.y; }
    int tot = 0;
#pragma unroll
    for (int ib = 0; ib < 8; ++ib) {
        const int4 ylo = lds128(a + (2 * ib) * 16), yhi = lds128(a + (2 * ib + 1) * 16);
        const int yl[4] = { ylo.x, ylo.y, ylo.z, ylo.w }, yh[4] = { yhi.x, yhi.y, yhi.z, yhi.w };
        int s = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            s = __dp4a((int)iq4nl_lookup4(ww[2 + 4 * ib + i]), yl[i], s);
            s = __dp4a((int)iq4nl_lookup4(ww[2 + 4 * ib + i] >> 4), yh[i], s);
        }
        tot += iq4xs_scale(ww[0], ww[1], ib) * s;
    }
    return (h2f(ww[0] & 0xFFFF) * *(const float *)(a + SB_OFF_D)) * (float)tot;
}

// Q4_1 / Q5_1 (block minimum m): the CPU backend pairs them with Q8_1 activations, whose s = fp16(d_unrounded * sum of the block's
// codes) multiplies m.  The eight s values of an act-task are expected as fp16 in the H32 slot of the record, which the Q8_0 family
// does not otherwise use (the in-kernel quantizer does not write them yet: these two dot products are host-verified only).
__device__ __forceinline__ void sb_load_q8_1_s(const uint8_t * a, float (&ys)[8]) {
    const int4 sv = lds128(a + SB_OFF_H32);
    const uint32_t u[4] = { (uint32_t)sv.x, (uint32_t)sv.y, (uint32_t)sv.z, (uint32_t)sv.w };
#pragma unroll
    for (int i = 0; i < 4; ++i) { ys[2 * i] = h2f(u[i] & 0xFFFF); ys[2 * i + 1] = h2f(u[i] >> 16); }
}
// Q4_1: task = 8 blocks of 20 bytes = 160 bytes; block = d | m (one word), 16 nibble bytes (four words)
template <> __device__ __forceinline__ float task_dot<T_Q4_1>(const uint8_t * w, const uint8_t * rec, int t) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
    uint32_t ww[40];
#pragma unroll
    for (int i = 0; i < 10; ++i) { const int4 v = lds128(w + 16 * i); ww[4 * i] = v.x; ww[4 * i + 1] = v.y; ww[4 * i + 2] = v.z; ww[4 * i + 3] = v.w; }
    const int4 da = lds128(a + SB_OFF_D), db = lds128(a + SB_OFF_D + 16);
    const float yd[8] = { __int_as_float(da.x), __int_as_float(da.y), __int_as_float(da.z), __int_as_float(da.w),
                          __int_as_float(db.x), __int_as_float(db.y), __int_as_float(db.z), __int_as_float(db.w) };
    float ys[8];
    sb_load_q8_1_s(a, ys);
    float acc = 0.0f;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
        const int4 ylo = lds128(a + (2 * b) * 16), yhi = lds128(a + (2 * b + 1) * 16);
        const int yl[4] = { ylo.x, ylo.y, ylo.z, ylo.w }, yh[4] = { yhi.x, yhi.y, yhi.z, yhi.w };
        int p0 = 0, p1 = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            p0 = __dp4a((int)(ww[5 * b + 1 + i] & 0x0F0F0F0F), yl[i], p0);
            p1 = dp4a_us(ww[5 * b + 1 + i] & 0xF0F0F0F0u, yh[i], p1);
        }
        acc += (h2f(ww[5 * b] & 0xFFFF) * yd[b]) * (float)(p0 + (p1 >> 4)) + h2f(ww[5 * b] >> 16) * ys[b];
    }
    return acc;
}
// Q5_1: task = 8 blocks of 24 bytes = 192 bytes; block = d | m, 32 fifth bits, 16 nibble bytes (six words)
template <> __device__ __forceinline__ float task_dot<T_Q5_1>(const uint8_t * w, const uint8_t * rec, int t) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
    uint32_t ww[48];
#pragma unroll
    for (int i = 0; i < 12; ++i) { const int4 v = lds128(w + 16 * i); ww[4 * i] = v.x; ww[4 * i + 1] = v.y; ww[4 * i + 2] = v.z; ww[4 * i + 3] = v.w; }
    const int4 da = lds128(a + SB_OFF_D), db = lds128(a + SB_OFF_D + 16);
    const float yd[8] = { __int_as_float(da.x), __int_as_float(da.y), __int_as_float(da.z), __int_as_float(da.w),
                          __int_as_float(db.x), __int_as_float(db.y), __int_as_float(db.z), __int_as_float(db.w) };
    float ys[8];
    sb_load_q8_1_s(a, ys);
    float acc = 0.0f;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
        const int4 ylo = lds128(a + (2 * b) * 16), yhi = lds128(a + (2 * b + 1) * 16);
        const int y[8] = { ylo.x, ylo.y, ylo.z, ylo.w, yhi.x, yhi.y, yhi.z, yhi.w };
        const uint32_t q[4] = { ww[6 * b + 2], ww[6 * b + 3], ww[6 * b + 4], ww[6 * b + 5] };
        const int s = q5_block_dot(q, ww[6 * b + 1], y);
        acc += (h2f(ww[6 * b] & 0xFFFF) * yd[b]) * (float)s + h2f(ww[6 * b] >> 16) * ys[b];
    }
    return acc;
}

// Q2_K: 84-byte superblocks are 4-byte aligned: 32-bit loads.  scales[16] (low nibble scale, high nibble min) words 0..3,
// qs words 4..19, d | dmin word 20.  Group g = 8 h + 2 j + l / 16 of the superblock = 16-value chunk g of the activations.
template <> __device__ __forceinline__ float task_dot<T_Q2_K>(const uint8_t * w, const uint8_t * rec, int t) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
    const uint32_t * wp = (const uint32_t *)w;
    const int4 sa = lds128(a + SB_OFF_S16), sb = lds128(a + SB_OFF_S16 + 16);
    const int s16w[8] = { sa.x, sa.y, sa.z, sa.w, sb.x, sb.y, sb.z, sb.w };       // sixteen 16-sums, int16 pairs
    int isum = 0, msum = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {                                                  // scale word k = groups 4k .. 4k+3
        const uint32_t scw = wp[k];
        const uint32_t mins = (scw >> 4) & 0x0F0F0F0Fu, scs = scw & 0x0F0F0F0Fu;
        msum = dp2a_lo_su(s16w[2 * k], mins, msum);
        msum = dp2a_hi_su(s16w[2 * k + 1], mins, msum);
#pragma unroll
        for (int gg = 0; gg < 4; ++gg) {
            const int g = 4 * k + gg, h = g >> 3, jj = (g >> 1) & 3, half16 = g & 1;
            const int4 yv = lds128(a + g * 16);
            const int y[4] = { yv.x, yv.y, yv.z, yv.w };
            int p = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) p = __dp4a((int)((wp[4 + 8 * h + 4 * half16 + i] >> (2 * jj)) & 0x03030303u), y[i], p);
            const int sc = gg == 0 ? ubyte<0>(scs) : gg == 1 ? ubyte<1>(scs) : gg == 2 ? ubyte<2>(scs) : ubyte<3>(scs);
            isum += sc * p;
        }
    }
    const float yd = *(const float *)(a + SB_OFF_D);
    const float dall = yd * h2f(wp[20] & 0xFFFF), dmin = yd * h2f(wp[20] >> 16);
    return dall * (float)isum - dmin * (float)msum;
}

// Q3_K: 110-byte superblocks are 2-byte aligned (as Q6_K): hmask words 0..7, qs words 8..23, scales words 24..26, d = low half of word 27
template <> __device__ __forceinline__ float task_dot<T_Q3_K>(const uint8_t * w, const uint8_t * rec, int t) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
    const uint32_t sh = ((uint32_t)(uintptr_t)w & 2) * 8;
    const uint32_t * wa = (const uint32_t *)((uintptr_t)w & ~(uintptr_t)3);
    auto word = [&](int i) { return __funnelshift_r(wa[i], wa[i + 1], sh); };
    // sixteen 6-bit scales (value - 32), four per word: low nibbles from bytes 0..7, two high bits each from bytes 8..11
    const uint32_t s0 = word(24), s1 = word(25), s2 = word(26);
    const uint32_t aux[4] = { ( s0       & 0x0F0F0F0Fu) | (( s2       & 0x03030303u) << 4),
                              ( s1       & 0x0F0F0F0Fu) | (((s2 >> 2) & 0x03030303u) << 4),
                              ((s0 >> 4) & 0x0F0F0F0Fu) | (((s2 >> 4) & 0x03030303u) << 4),
                              ((s1 >> 4) & 0x0F0F0F0Fu) | (((s2 >> 6) & 0x03030303u) << 4) };
    int isum = 0;
#pragma unroll
    for (int g = 0; g < 16; ++g) {
        const int h = g >> 3, jj = (g >> 1) & 3, half16 = g & 1, bit = 4 * h + jj;
        const int4 yv = lds128(a + g * 16);
        const int y[4] = { yv.x, yv.y, yv.z, yv.w };
        int p = 0, low = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            p   = __dp4a((int)((word(8 + 8 * h + 4 * half16 + i) >> (2 * jj)) & 0x03030303u), y[i], p);
            low = __dp4a((int)(~(word(4 * half16 + i) >> bit) & 0x01010101u), y[i], low);        // activations whose high bit is clear
        }
        const uint32_t ax = aux[g >> 2];
        const int sc = ((g & 3) == 0 ? ubyte<0>(ax) : (g & 3) == 1 ? ubyte<1>(ax) : (g & 3) == 2 ? ubyte<2>(ax) : ubyte<3>(ax)) - 32;
        isum += sc * (p - 4 * low);
    }
    return (h2f(word(27) & 0xFFFF) * *(const float *)(a + SB_OFF_D)) * (float)isum;
}

// ----------------------------------------------------------------------------- two rows against one activation task
// Round-2 experiment, host-verified only (not dispatched): the same lane dots task t of TWO weight rows, so every activation chunk
// is read from shared memory once instead of twice (activation reads are about half of the kernel's shared-memory
// traffic).  Per row the operations are those of q45_task, so results are bit-identical to task_dot.
template <int C, bool FIVE>
__device__ __forceinline__ void q45_chunk2(const uint8_t * qs0, const uint8_t * qs1, const uint32_t (&qh0)[8], const uint32_t (&qh1)[8], const uint8_t * a,
                                            int sa0, int sa1, int sb0, int sb1, int & acc0, int & acc1) {
    const int4 qa0 = lds128(qs0 + 32 * C), qb0 = lds128(qs0 + 32 * C + 16), qa1 = lds128(qs1 + 32 * C), qb1 = lds128(qs1 + 32 * C + 16);
    const uint32_t q0[8] = { (uint32_t)qa0.x, (uint32_t)qa0.y, (uint32_t)qa0.z, (uint32_t)qa0.w, (uint32_t)qb0.x, (uint32_t)qb0.y, (uint32_t)qb0.z, (uint32_t)qb0.w };
    const uint32_t q1[8] = { (uint32_t)qa1.x, (uint32_t)qa1.y, (uint32_t)qa1.z, (uint32_t)qa1.w, (uint32_t)qb1.x, (uint32_t)qb1.y, (uint32_t)qb1.z, (uint32_t)qb1.w };
    int p00 = 0, p01 = 0, p10 = 0, p11 = 0;                       // p<row><low/high sub-block>
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int4 ylo = lds128(a + (4 * C + h) * 16), yhi = lds128(a + (4 * C + 2 + h) * 16);
        const int yl[4] = { ylo.x, ylo.y, ylo.z, ylo.w }, yh[4] = { yhi.x, yhi.y, yhi.z, yhi.w };
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t x0 = q0[4 * h + i], x1 = q1[4 * h + i];
            if constexpr (FIVE) {
                const uint32_t h0 = qh0[4 * h + i] >> (2 * C), h1 = qh1[4 * h + i] >> (2 * C);
                p00 = __dp4a((int)((x0 & 0x0F0F0F0F) | ((h0 & 0x01010101) << 4)), yl[i], p00);
                p01 = __dp4a((int)(((x0 >> 4) & 0x0F0F0F0F) | ((h0 & 0x02020202) << 3)), yh[i], p01);
                p10 = __dp4a((int)((x1 & 0x0F0F0F0F) | ((h1 & 0x01010101) << 4)), yl[i], p10);
                p11 = __dp4a((int)(((x1 >> 4) & 0x0F0F0F0F) | ((h1 & 0x02020202) << 3)), yh[i], p11);
            } else {
                p00 = __dp4a((int)(x0 & 0x0F0F0F0F), yl[i], p00);
                p01 = dp4a_us(x0 & 0xF0F0F0F0u, yh[i], p01);
                p10 = __dp4a((int)(x1 & 0x0F0F0F0F), yl[i], p10);
                p11 = dp4a_us(x1 & 0xF0F0F0F0u, yh[i], p11);
            }
        }
    }
    if constexpr (!FIVE) { p01 >>= 4; p11 >>= 4; }
    acc0 += sa0 * p00 + sb0 * p01;
    acc1 += sa1 * p10 + sb1 * p11;
}

template <bool FIVE> __device__ __forceinline__ void q45_task2(const uint8_t * w0, const uint8_t * w1, const uint8_t * rec, int t, float & r0, float & r1) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
    const int4 hdr0 = lds128(w0), hdr1 = lds128(w1);
    const int4 h32 = lds128(a + SB_OFF_H32);
    uint32_t qh0[8] = { 0, 0, 0, 0, 0, 0, 0, 0 }, qh1[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    if constexpr (FIVE) {
        const int4 a0 = lds128(w0 + 16), b0 = lds128(w0 + 32), a1 = lds128(w1 + 16), b1 = lds128(w1 + 32);
        qh0[0] = a0.x; qh0[1] = a0.y; qh0[2] = a0.z; qh0[3] = a0.w; qh0[4] = b0.x; qh0[5] = b0.y; qh0[6] = b0.z; qh0[7] = b0.w;
        qh1[0] = a1.x; qh1[1] = a1.y; qh1[2] = a1.z; qh1[3] = a1.w; qh1[4] = b1.x; qh1[5] = b1.y; qh1[6] = b1.z; qh1[7] = b1.w;
    }
    const uint8_t * qs0 = w0 + (FIVE ? 48 : 16), * qs1 = w1 + (FIVE ? 48 : 16);
    int accs[2] = { 0, 0 }, accm[2];
    uint32_t sc_lo[2], sc_hi[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int4 & hdr = r == 0 ? hdr0 : hdr1;
        const uint32_t s0 = hdr.y, s1 = hdr.z, s2 = hdr.w;
        const uint32_t mn_lo = s1 & 0x3F3F3F3Fu, mn_hi = ((s2 >> 4) & 0x0F0F0F0Fu) | ((s1 >> 2) & 0x30303030u);
        sc_lo[r] = s0 & 0x3F3F3F3Fu;
        sc_hi[r] = (s2 & 0x0F0F0F0Fu) | ((s0 >> 2) & 0x30303030u);
        int m = dp2a_lo_su(h32.x, mn_lo, 0);
        m = dp2a_hi_su(h32.y, mn_lo, m);
        m = dp2a_lo_su(h32.z, mn_hi, m);
        m = dp2a_hi_su(h32.w, mn_hi, m);
        accm[r] = m;
    }
    q45_chunk2<0, FIVE>(qs0, qs1, qh0, qh1, a, ubyte<0>(sc_lo[0]), ubyte<0>(sc_lo[1]), ubyte<1>(sc_lo[0]), ubyte<1>(sc_lo[1]), accs[0], accs[1]);
    q45_chunk2<1, FIVE>(qs0, qs1, qh0, qh1, a, ubyte<2>(sc_lo[0]), ubyte<2>(sc_lo[1]), ubyte<3>(sc_lo[0]), ubyte<3>(sc_lo[1]), accs[0], accs[1]);
    q45_chunk2<2, FIVE>(qs0, qs1, qh0, qh1, a, ubyte<0>(sc_hi[0]), ubyte<0>(sc_hi[1]), ubyte<1>(sc_hi[0]), ubyte<1>(sc_hi[1]), accs[0], accs[1]);
    q45_chunk2<3, FIVE>(qs0, qs1, qh0, qh1, a, ubyte<2>(sc_hi[0]), ubyte<2>(sc_hi[1]), ubyte<3>(sc_hi[0]), ubyte<3>(sc_hi[1]), accs[0], accs[1]);
    const float yd = *(const float *)(a + SB_OFF_D);
    {
        const float d = h2f((uint32_t)hdr0.x & 0xFFFF) * yd, dmin = h2f((uint32_t)hdr0.x >> 16) * yd;
        r0 = d * (float)accs[0] - dmin * (float)accm[0];
    }
    {
        const float d = h2f((uint32_t)hdr1.x & 0xFFFF) * yd, dmin = h2f((uint32_t)hdr1.x >> 16) * yd;
        r1 = d * (float)accs[1] - dmin * (float)accm[1];
    }
}

// ----------------------------------------------------------------------------- activation-stationary form (Q4_K / Q5_K, n = 1, K <= 4096)
// With at most 16 tasks per row one warp covers a whole row, so a lane's task is the same in every row of the launch.  Lanes 2t and
// 2t+1 own task t (superblock t of every row); lane 2t + h takes its 64-weight chunks 2h and 2h+1, with the sub-block scales and mins
// of sc_lo / mn_lo (h = 0) or sc_hi / mn_hi (h = 1).  Each lane loads its half of act-task t from the shared record into registers
// once (32 code words, two h32 words, the scale) and from then on reads only weights from shared memory.
// The halves' integer sums are added with an xor-1 shuffle before the f32 scaling, so each task's float is the one q45_task returns,
// and the row is reduced over lanes xor 16, 8, 4, 2: the tree of the task-per-lane kernel (xor 8, 4, 2, 1 over task indices).
// The result is bit-identical to the task-per-lane kernel's, and so to column c of the n-column kernel.
struct q45_acts {
    int y[32];       // codes 128 h .. 128 h + 127 of act-task t
    int h32[2];      // the 32-sums of sub-blocks 4h .. 4h + 3, int16 pairs
    float d;         // the act-task's scale
};
__device__ __forceinline__ void q45_load_acts(const uint8_t * rec, int t, int h, q45_acts & A) {
    const uint8_t * a = rec + (size_t)t * SB_REC;
#pragma unroll
    for (int i = 0; i < 8; ++i) { const int4 v = lds128(a + 128 * h + 16 * i); A.y[4 * i] = v.x; A.y[4 * i + 1] = v.y; A.y[4 * i + 2] = v.z; A.y[4 * i + 3] = v.w; }
    const uint2 hv = *(const uint2 *)(a + SB_OFF_H32 + 8 * h);
    A.h32[0] = (int)hv.x; A.h32[1] = (int)hv.y;
    A.d = *(const float *)(a + SB_OFF_D);
}

// chunk C (0, 1) of this lane's half: q45_chunk with the activations taken from registers (qh already shifted by 4h)
template <int C, bool FIVE>
__device__ __forceinline__ void q45_chunk_regs(const uint8_t * qs, const uint32_t (&qh)[8], const int (&y)[32], int sc0, int sc1, int & acc_s) {
    const int4 qa = lds128(qs + 32 * C), qb = lds128(qs + 32 * C + 16);
    const uint32_t q[8] = { (uint32_t)qa.x, (uint32_t)qa.y, (uint32_t)qa.z, (uint32_t)qa.w, (uint32_t)qb.x, (uint32_t)qb.y, (uint32_t)qb.z, (uint32_t)qb.w };
    int p0 = 0, p1 = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t qq = q[4 * h + i];
            const int yl = y[16 * C + 4 * h + i], yh = y[16 * C + 8 + 4 * h + i];
            if constexpr (FIVE) {
                const uint32_t hb = qh[4 * h + i] >> (2 * C);
                p0 = __dp4a((int)((qq & 0x0F0F0F0F) | ((hb & 0x01010101) << 4)), yl, p0);
                p1 = __dp4a((int)(((qq >> 4) & 0x0F0F0F0F) | ((hb & 0x02020202) << 3)), yh, p1);
            } else {
                p0 = __dp4a((int)(qq & 0x0F0F0F0F), yl, p0);
                p1 = dp4a_us(qq & 0xF0F0F0F0u, yh, p1);
            }
        }
    }
    if constexpr (!FIVE) p1 >>= 4;
    acc_s += sc0 * p0 + sc1 * p1;
}

// this lane's half of task t of one row (w = the task's first byte): integer sums and the task's d | dmin word
template <bool FIVE> __device__ __forceinline__ void q45_half_regs(const uint8_t * w, const q45_acts & A, int h, int & acc_s, int & acc_m, uint32_t & dm) {
    const int4 hdr = lds128(w);                                         // d | dmin | scales[12]
    uint32_t qh[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    if constexpr (FIVE) {
        const int4 ha = lds128(w + 16), hb = lds128(w + 32);
        const uint32_t raw[8] = { (uint32_t)ha.x, (uint32_t)ha.y, (uint32_t)ha.z, (uint32_t)ha.w, (uint32_t)hb.x, (uint32_t)hb.y, (uint32_t)hb.z, (uint32_t)hb.w };
#pragma unroll
        for (int i = 0; i < 8; ++i) qh[i] = raw[i] >> (4 * h);
    }
    const uint8_t * qs = w + (FIVE ? 48 : 16) + 64 * h;
    const uint32_t s0 = hdr.y, s1 = hdr.z, s2 = hdr.w;
    const uint32_t sc = h ? ((s2 & 0x0F0F0F0Fu) | ((s0 >> 2) & 0x30303030u)) : (s0 & 0x3F3F3F3Fu);
    const uint32_t mn = h ? (((s2 >> 4) & 0x0F0F0F0Fu) | ((s1 >> 2) & 0x30303030u)) : (s1 & 0x3F3F3F3Fu);
    acc_m = dp2a_lo_su(A.h32[0], mn, 0);
    acc_m = dp2a_hi_su(A.h32[1], mn, acc_m);
    acc_s = 0;
    q45_chunk_regs<0, FIVE>(qs, qh, A.y, ubyte<0>(sc), ubyte<1>(sc), acc_s);
    q45_chunk_regs<1, FIVE>(qs, qh, A.y, ubyte<2>(sc), ubyte<3>(sc), acc_s);
    dm = (uint32_t)hdr.x;
}

// R rows (a power of two, mmvq_sb.cu takes 2; row j's first byte at row[j]) against the activations.  All 32 lanes call this together; lanes whose task is
// beyond the row (t >= ntasks) contribute 0, as idle lanes of the task-per-lane kernel do.  Row j's dot product is returned in lanes
// 32 j / R .. 32 (j + 1) / R - 1.  While rows remain to be split, a reduction step exchanges rows (a lane keeps the rows of its side of
// the xor distance and sends the others), so R rows cost one shuffle per row and step at most, and each row is still summed by the
// tree xor 16, 8, 4, 2.
template <bool FIVE, int R> __device__ __forceinline__ float q45_rows_regs(const uint8_t * const (&row)[R], const q45_acts & A, int lane, int ntasks) {
    const int t = lane >> 1, h = lane & 1;
    int s[R], m[R];
    uint32_t dm[R];
#pragma unroll
    for (int j = 0; j < R; ++j) { s[j] = 0; m[j] = 0; dm[j] = 0; }
    if (t < ntasks) {
#pragma unroll
        for (int j = 0; j < R; ++j) q45_half_regs<FIVE>(row[j] + (size_t)t * (FIVE ? 176 : 144), A, h, s[j], m[j], dm[j]);
    }
    float x[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
        s[j] += __shfl_xor_sync(0xffffffffu, s[j], 1);                 // integer sums of the whole task: exact
        m[j] += __shfl_xor_sync(0xffffffffu, m[j], 1);
        x[j] = 0.0f;
        if (t < ntasks) {
            const float d = h2f(dm[j] & 0xFFFF) * A.d, dmin = h2f(dm[j] >> 16) * A.d;
            x[j] += d * (float)s[j] - dmin * (float)m[j];
        }
    }
#pragma unroll
    for (int n = R, o = 16; o > 1; o >>= 1) {
        if (n > 1) {
            const bool up = (lane & o) != 0;
#pragma unroll
            for (int j = 0; j < n / 2; ++j) {
                const float keep = up ? x[n / 2 + j] : x[j], send = up ? x[j] : x[n / 2 + j];
                x[j] = keep + __shfl_xor_sync(0xffffffffu, send, o);
            }
            n /= 2;
        } else {
            x[0] += __shfl_xor_sync(0xffffffffu, x[0], o);
        }
    }
    return x[0];
}

// ----------------------------------------------------------------------------- several activation columns (2 <= n <= 8)
// The weights of a task are decoded once and dotted with every column's record (records of column c at rec + c * rec_stride).
// Per column the floating-point operations are exactly those of the n = 1 path, so column c of an n-column product is
// bit-identical to the n = 1 product with that column.
template <int C, bool FIVE, int NC>
__device__ __forceinline__ void q45_chunk_nc(const uint8_t * qs, const uint32_t (&qh)[8], const uint8_t * a0, int rec_stride, int ncols, int sc0, int sc1, int (&acc_s)[NC]) {
    const int4 qa = lds128(qs + 32 * C), qb = lds128(qs + 32 * C + 16);
    const uint32_t q[8] = { (uint32_t)qa.x, (uint32_t)qa.y, (uint32_t)qa.z, (uint32_t)qa.w, (uint32_t)qb.x, (uint32_t)qb.y, (uint32_t)qb.z, (uint32_t)qb.w };
    uint32_t lo[8], hi[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        if constexpr (FIVE) {
            const uint32_t hb = qh[i] >> (2 * C);
            lo[i] = (q[i] & 0x0F0F0F0F) | ((hb & 0x01010101) << 4);
            hi[i] = ((q[i] >> 4) & 0x0F0F0F0F) | ((hb & 0x02020202) << 3);
        } else {
            lo[i] = q[i] & 0x0F0F0F0F;
            hi[i] = q[i] & 0xF0F0F0F0u;                                               // 16 x the high nibbles
        }
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        if (c < ncols) {
            const uint8_t * a = a0 + c * rec_stride;
            int p0 = 0, p1 = 0;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int4 ylo = lds128(a + (4 * C + h) * 16), yhi = lds128(a + (4 * C + 2 + h) * 16);
                const int yl[4] = { ylo.x, ylo.y, ylo.z, ylo.w }, yh[4] = { yhi.x, yhi.y, yhi.z, yhi.w };
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    p0 = __dp4a((int)lo[4 * h + i], yl[i], p0);
                    if constexpr (FIVE) p1 = __dp4a((int)hi[4 * h + i], yh[i], p1);
                    else                p1 = dp4a_us(hi[4 * h + i], yh[i], p1);
                }
            }
            if constexpr (!FIVE) p1 >>= 4;
            acc_s[c] += sc0 * p0 + sc1 * p1;
        }
    }
}

template <bool FIVE, int NC>
__device__ __forceinline__ void q45_task_nc(const uint8_t * w, const uint8_t * rec, int rec_stride, int t, int ncols, float (&acc)[NC]) {
    const uint8_t * a0 = rec + (size_t)t * SB_REC;
    const int4 hdr = lds128(w);
    uint32_t qh[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    if constexpr (FIVE) {
        const int4 ha = lds128(w + 16), hb = lds128(w + 32);
        qh[0] = ha.x; qh[1] = ha.y; qh[2] = ha.z; qh[3] = ha.w; qh[4] = hb.x; qh[5] = hb.y; qh[6] = hb.z; qh[7] = hb.w;
    }
    const uint8_t * qs = w + (FIVE ? 48 : 16);
    const uint32_t s0 = hdr.y, s1 = hdr.z, s2 = hdr.w;
    const uint32_t sc_lo = s0 & 0x3F3F3F3Fu, mn_lo = s1 & 0x3F3F3F3Fu;
    const uint32_t sc_hi = (s2 & 0x0F0F0F0Fu) | ((s0 >> 2) & 0x30303030u);
    const uint32_t mn_hi = ((s2 >> 4) & 0x0F0F0F0Fu) | ((s1 >> 2) & 0x30303030u);
    int acc_s[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) acc_s[c] = 0;
    q45_chunk_nc<0, FIVE, NC>(qs, qh, a0, rec_stride, ncols, ubyte<0>(sc_lo), ubyte<1>(sc_lo), acc_s);
    q45_chunk_nc<1, FIVE, NC>(qs, qh, a0, rec_stride, ncols, ubyte<2>(sc_lo), ubyte<3>(sc_lo), acc_s);
    q45_chunk_nc<2, FIVE, NC>(qs, qh, a0, rec_stride, ncols, ubyte<0>(sc_hi), ubyte<1>(sc_hi), acc_s);
    q45_chunk_nc<3, FIVE, NC>(qs, qh, a0, rec_stride, ncols, ubyte<2>(sc_hi), ubyte<3>(sc_hi), acc_s);
    const float wd = h2f((uint32_t)hdr.x & 0xFFFF), wm = h2f((uint32_t)hdr.x >> 16);
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        if (c < ncols) {
            const uint8_t * a = a0 + c * rec_stride;
            const int4 h32 = lds128(a + SB_OFF_H32);
            int acc_m = dp2a_lo_su(h32.x, mn_lo, 0);
            acc_m = dp2a_hi_su(h32.y, mn_lo, acc_m);
            acc_m = dp2a_lo_su(h32.z, mn_hi, acc_m);
            acc_m = dp2a_hi_su(h32.w, mn_hi, acc_m);
            const float yd = *(const float *)(a + SB_OFF_D);
            const float d = wd * yd, dmin = wm * yd;
            acc[c] += d * (float)acc_s[c] - dmin * (float)acc_m;
        }
    }
}

template <int T, int NC>
__device__ __forceinline__ void task_dot_nc(const uint8_t * w, const uint8_t * rec, int rec_stride, int t, int ncols, float (&acc)[NC]) {
    if constexpr (T == T_Q4_K)      q45_task_nc<false, NC>(w, rec, rec_stride, t, ncols, acc);
    else if constexpr (T == T_Q5_K) q45_task_nc<true, NC>(w, rec, rec_stride, t, ncols, acc);
    else {
        // other formats: the single-column dot product per column (the weight bytes are re-read from shared memory, not from HBM)
#pragma unroll
        for (int c = 0; c < NC; ++c) if (c < ncols) acc[c] += task_dot<T>(w, rec + c * rec_stride, t);
    }
}

} // namespace b200
