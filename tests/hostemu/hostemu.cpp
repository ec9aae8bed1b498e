// hostemu.cpp — TEST INFRASTRUCTURE ONLY: the per-thread decode logic of ggml_b200/csrc (unit dot products, element decoders)
// compiled for the host through tests/hostemu/shim, exported with a C ABI for tests/test_hostemu_kernel_logic.py.
// It checks indexing / bit manipulation of the block formats on the CPU; it says nothing about scheduling, memory movement or
// the PTX-level instructions (dp2a, prmt, wgmma ...) of the fast kernels — those are covered by the `-m gpu` parity tests.
#define B200_HOST_EMU 1
#include "cuda_shim.h"
#include <vector>
#include "../../ggml_b200/csrc/b200_dequant.cuh"
#include "../../ggml_b200/csrc/b200_sb_tasks.cuh"
#include "../../ggml_b200/csrc/b200_tc_dequant.cuh"
#include "../../ggml_b200/csrc/b200_sb_mma.cuh"

using namespace b200;

template <int T> static float row_dot(const uint8_t * row, int64_t K, const uint8_t * rec) {
    const act_layout L = make_act_layout(K, fmt<T>::ACT_K != 0);
    float acc = 0.0f;
    for (int u = 0; u < (int)(K / 64); ++u) {
        unit_act A;
        load_unit_act<T>(rec, L, u, A);
        acc += unit_dot<T>(row, u, A);
    }
    if constexpr (fmt<T>::QK == 32) {                       // odd number of 32-blocks: the kernels' trailing-block path
        const int nunits = (int)(K / 64);
        if ((K & 63) != 0) acc += tail_block_dot<T>(row + (size_t)nunits * 2 * fmt<T>::BYTES, rec, L, nunits * 2);
    }
    return acc;
}
template <int T> static void dequant_all(const uint8_t * src, float * dst, int64_t n) {
    for (int64_t e = 0; e < n; e += 4) { float o[4]; dequant4<T>(src, e, o); for (int i = 0; i < 4; ++i) dst[e + i] = o[i]; }
}

#define FOR_TYPES(X) X(T_Q4_0) X(T_Q8_0) X(T_Q4_K) X(T_Q5_K) X(T_Q6_K) X(T_Q4_1) X(T_Q5_0) X(T_Q5_1) X(T_Q2_K) X(T_Q3_K) X(T_IQ4_NL) X(T_IQ4_XS) X(T_IQ2_XXS) X(T_IQ3_XXS) X(T_IQ1_S) X(T_IQ2_XS) X(T_IQ2_S) X(T_IQ3_S) X(T_IQ1_M) X(T_TQ1_0) X(T_TQ2_0)

// tensor-core GEMM operand preparation: one W row -> K fp16 values (swizzle key 0: the 8 chunks of a K-step land in order)
template <int T> static void tc_row(const uint8_t * row, int64_t K, uint16_t * out) {
    constexpr int UK = tcfmt<T>::UNIT_KSTEPS, UW = tcfmt<T>::UNIT_WORDS;
    const int64_t nunits = K / (64 * UK);
    const size_t unit_bytes = (size_t)row_bytes(T, 64 * UK);
    for (int64_t u = 0; u < nunits; ++u) {
        uint32_t regs[UW];
        tc_load_unit<T>(row + u * unit_bytes, regs);
        uint8_t * dst = (uint8_t *)(out + (u * UK) * 64);
        dq64<T, 0>(regs, dst, 0);
        dq64<T, 1>(regs, dst + 128, 0);
        if constexpr (UK == 4) { dq64<T, 2>(regs, dst + 256, 0); dq64<T, 3>(regs, dst + 384, 0); }
    }
}

template <int T> static float sb_row(const uint8_t * row, int64_t K, const uint8_t * rec) {
    float acc = 0.0f;
    for (int t = 0; t < (int)(K / sbfmt<T>::TASK_W); ++t) acc += task_dot<T>(row + (size_t)t * sbfmt<T>::TASK_B, rec, t);
    return acc;
}
template <int T> static void sb_row_nc(const uint8_t * row, int64_t K, const uint8_t * rec, int rec_stride, int ncols, float * out) {
    float acc[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    for (int t = 0; t < (int)(K / sbfmt<T>::TASK_W); ++t) task_dot_nc<T, 8>(row + (size_t)t * sbfmt<T>::TASK_B, rec, rec_stride, t, ncols, acc);
    for (int c = 0; c < 8; ++c) out[c] = acc[c];
}
// ---- the mma small-batch consume path (b200_sb_mma.cuh): one emulated warp, a tile of 16 packed rows (row r at rows + r * pitch) against
// ncols (<= 8) activation columns (column c at x + c * K): planar records by the kernel's quantizer, every task by mma_task; out[16][8]
template <int T> static void mma_tile(const uint8_t * rows, int64_t pitch, int64_t K, const float * x, int ncols, float * out) {
    using F = mmafmt<T>;
    const mma_act A = make_mma_act(K, F::KQ, F::S16, F::RESIDUE, mma_s81<T>::value);
    std::vector<uint8_t> rec((size_t)ncols * A.col_bytes + 64);
    uint8_t * recp = rec.data();
    warp_emu::run([&] {
        const int lane = (int)(threadIdx.x & 31);
        for (int i0 = 0; i0 < ncols * A.ntask; i0 += 2) {
            const int i = i0 + (lane >> 4);
            const bool ok = i < ncols * A.ntask;
            const int c = ok ? i / A.ntask : 0, t = ok ? i % A.ntask : 0;
            mma_quantize_task_h<F::KQ, F::S16, mma_s81<T>::value>(x + (size_t)c * K, ok, recp + (size_t)c * A.col_bytes, A, t);
        }
        pthread_barrier_wait(&warp_emu::barrier());
        const int g = lane >> 2, t = lane & 3;
        mma_cols C;
        C.b  = recp + (size_t)std::min(g, ncols - 1) * A.col_bytes;
        C.c0 = recp + (size_t)std::min(2 * t, ncols - 1) * A.col_bytes;
        C.c1 = recp + (size_t)std::min(2 * t + 1, ncols - 1) * A.col_bytes;
        float facc[4] = { 0, 0, 0, 0 };
        for (int task = 0; task < (int)(K / 256); ++task)
            mma_task<T>(rows + (size_t)g * pitch + (size_t)task * F::TASK_B, rows + (size_t)(g + 8) * pitch + (size_t)task * F::TASK_B, C, A, task, t, facc);
        out[(size_t)g * 8 + 2 * t] = facc[0]; out[(size_t)g * 8 + 2 * t + 1] = facc[1];
        out[(size_t)(g + 8) * 8 + 2 * t] = facc[2]; out[(size_t)(g + 8) * 8 + 2 * t + 1] = facc[3];
    });
}
extern "C" {

// offsets of the activation record sections: out = { off_bs, off_d, off_s (or -1), bytes }
void emu_act_layout(int64_t K, int kq, int32_t * out) {
    const act_layout L = make_act_layout(K, kq != 0);
    out[0] = L.off_bs; out[1] = L.off_d; out[2] = -1; out[3] = L.bytes;
#ifdef B200_ACT_HAS_S
    out[2] = L.off_s;
#endif
}
int emu_type_is_kquant(int type) { return type_is_kquant(type) ? 1 : 0; }
int64_t emu_row_bytes(int type, int64_t K) { return (int64_t)row_bytes(type, K); }

// dot product of one packed weight row with one activation record (K % 32 == 0 for 32-block formats, else K % 256 == 0)
float emu_row_dot(int type, const uint8_t * row, int64_t K, const uint8_t * rec) {
    switch (type) {
#define X(T) case T: return row_dot<T>(row, K, rec);
        FOR_TYPES(X)
#undef X
        default: return NAN;
    }
}
int emu_dequant(int type, const uint8_t * src, float * dst, int64_t n) {
    switch (type) {
#define X(T) case T: dequant_all<T>(src, dst, n); return 0;
        FOR_TYPES(X)
#undef X
        default: return -1;
    }
}

// ---- activation quantizers, one emulated warp (32 host threads in lockstep; shuffles = exchanges between barriers)
// generic-path record (q | bs | d | s): quantize_act_kernel's cta_quantize_row with a one-warp CTA
int emu_quantize_record(int kq, const float * x, int64_t K, uint8_t * rec) {
    const act_layout L = make_act_layout(K, kq != 0);
    warp_emu::run([&] { if (kq) cta_quantize_row<true>(x, K, rec, L); else cta_quantize_row<false>(x, K, rec, L); });
    return L.bytes;
}
// superblock-kernel records (SB_REC bytes per act-task): the kernel's quantization loop for one column, one warp
int emu_sb_quantize(int kq, const float * x, int64_t K, uint8_t * rec, int with_q8_1_s) {
    const int ntask = (int)(K / 256);
    warp_emu::run([&] {
        const int lane = (int)(threadIdx.x & 31);
        for (int i0 = 0; i0 < ntask; i0 += 2) {
            const int t = i0 + (lane >> 4);
            const bool ok = t < ntask;
            if (kq) sb_quantize_task_h<true>(x, ok, rec, ok ? t : 0);
            else if (with_q8_1_s) sb_quantize_task_h<false, true>(x, ok, rec, ok ? t : 0);
            else sb_quantize_task_h<false>(x, ok, rec, ok ? t : 0);
        }
    });
    return ntask * SB_REC;
}

// ---- GEMM operand preparation (b200_tc_dequant.cuh): K fp16 values of one packed row
#define FOR_TC_TYPES(X) X(T_Q4_0) X(T_Q8_0) X(T_Q4_K) X(T_Q5_K) X(T_Q6_K) X(T_Q4_1) X(T_Q5_0) X(T_Q5_1) X(T_IQ4_NL) X(T_IQ4_XS) X(T_Q2_K) X(T_Q3_K)
int emu_tc_dequant_row(int type, const uint8_t * row, int64_t K, uint16_t * out) {
    switch (type) {
#define X(T) case T: tc_row<T>(row, K, out); return 0;
        FOR_TC_TYPES(X)
#undef X
        default: return -1;
    }
}

// ---- the superblock mat-vec kernel's per-lane task dot products (b200_sb_tasks.cuh); hot-path formats only
#define FOR_SB_TYPES(X) X(T_Q4_0) X(T_Q8_0) X(T_Q4_K) X(T_Q5_K) X(T_Q6_K) X(T_Q5_0) X(T_Q2_K) X(T_Q3_K) X(T_Q4_1) X(T_Q5_1) X(T_IQ4_NL) X(T_IQ4_XS)
// out = { TASK_W, TASK_B, SB_REC, SB_OFF_S32, SB_OFF_S16, SB_OFF_H32, SB_OFF_D }
int emu_sb_geometry(int type, int32_t * out) {
    switch (type) {
#define X(T) case T: out[0] = sbfmt<T>::TASK_W; out[1] = sbfmt<T>::TASK_B; break;
        FOR_SB_TYPES(X)
#undef X
        default: return -1;
    }
    out[2] = SB_REC; out[3] = SB_OFF_S32; out[4] = SB_OFF_S16; out[5] = SB_OFF_H32; out[6] = SB_OFF_D;
    return 0;
}
// two rows sharing the activation loads (Q4_K / Q5_K): out[0], out[1]
int emu_sb_two_row_dot(int type, const uint8_t * row0, const uint8_t * row1, int64_t K, const uint8_t * rec, float * out) {
    float a0 = 0.0f, a1 = 0.0f;
    for (int t = 0; t < (int)(K / 256); ++t) {
        float r0, r1;
        if (type == T_Q4_K)      q45_task2<false>(row0 + (size_t)t * 144, row1 + (size_t)t * 144, rec, t, r0, r1);
        else if (type == T_Q5_K) q45_task2<true>(row0 + (size_t)t * 176, row1 + (size_t)t * 176, rec, t, r0, r1);
        else return -1;
        a0 += r0; a1 += r1;
    }
    out[0] = a0; out[1] = a1;
    return 0;
}
float emu_sb_row_dot(int type, const uint8_t * row, int64_t K, const uint8_t * rec) {
    switch (type) {
#define X(T) case T: return sb_row<T>(row, K, rec);
        FOR_SB_TYPES(X)
#undef X
        default: return NAN;
    }
}
int emu_sb_row_dot_nc(int type, const uint8_t * row, int64_t K, const uint8_t * rec, int rec_stride, int ncols, float * out) {
    switch (type) {
#define X(T) case T: sb_row_nc<T>(row, K, rec, rec_stride, ncols, out); return 0;
        FOR_SB_TYPES(X)
#undef X
        default: return -1;
    }
}

int emu_mma_tile(int type, const uint8_t * rows, int64_t pitch, int64_t K, const float * x, int ncols, float * out) {
    switch (type) {
        case T_Q4_0: mma_tile<T_Q4_0>(rows, pitch, K, x, ncols, out); return 0;
        case T_Q8_0: mma_tile<T_Q8_0>(rows, pitch, K, x, ncols, out); return 0;
        case T_Q4_K: mma_tile<T_Q4_K>(rows, pitch, K, x, ncols, out); return 0;
        case T_Q5_K: mma_tile<T_Q5_K>(rows, pitch, K, x, ncols, out); return 0;
        case T_Q6_K: mma_tile<T_Q6_K>(rows, pitch, K, x, ncols, out); return 0;
        case T_Q5_0: mma_tile<T_Q5_0>(rows, pitch, K, x, ncols, out); return 0;
        case T_Q4_1: mma_tile<T_Q4_1>(rows, pitch, K, x, ncols, out); return 0;
        case T_Q5_1: mma_tile<T_Q5_1>(rows, pitch, K, x, ncols, out); return 0;
        case T_IQ4_NL: mma_tile<T_IQ4_NL>(rows, pitch, K, x, ncols, out); return 0;
        case T_IQ4_XS: mma_tile<T_IQ4_XS>(rows, pitch, K, x, ncols, out); return 0;
        case T_Q2_K: mma_tile<T_Q2_K>(rows, pitch, K, x, ncols, out); return 0;
        case T_Q3_K: mma_tile<T_Q3_K>(rows, pitch, K, x, ncols, out); return 0;
        default: return -1;
    }
}

} // extern "C"
