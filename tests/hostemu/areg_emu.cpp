// areg_emu.cpp — TEST INFRASTRUCTURE ONLY.  The activation-stationary consume form of mmvq_sb.cu (q45_load_acts / q45_rows_regs,
// b200_sb_tasks.cuh) in one emulated warp (32 host threads in lockstep, shuffles through tests/hostemu/shim), beside the task-per-lane
// consume it replaces for Q4_K / Q5_K at n = 1, so that the CPU-only suite can check the two bit for bit.
#define B200_HOST_EMU 1
#include "cuda_shim.h"
#include "../../ggml_b200/csrc/b200_sb_tasks.cuh"

using namespace b200;

// the kernel's row loop of the activation-stationary form, one warp: R rows per pass, rows past the end repeat the last one
template <int T, int R> static void rows_regs(const uint8_t * rows, int nrows, size_t rb, const q45_acts & A, int lane, int ntasks, float * out, float * lanes) {
    for (int r0 = 0; r0 < nrows; r0 += R) {
        const uint8_t * rp[R];
        for (int j = 0; j < R; ++j) rp[j] = rows + (size_t)std::min(r0 + j, nrows - 1) * rb;
        const float v = q45_rows_regs<T == T_Q5_K, R>(rp, A, lane, ntasks);
        const int r = r0 + lane / (32 / R);
        if (r < nrows) lanes[(size_t)r * 32 + lane % (32 / R)] = v;
        if (lane % (32 / R) == 0 && r < nrows) out[r] = v;
    }
}

template <int T>
static void rows_both(const uint8_t * rows, int nrows, int64_t K, const float * x, uint8_t * rec, float * out_regs, float * out_lanes, float * out_tasks) {
    constexpr int TB = sbfmt<T>::TASK_B, LPR = sbfmt<T>::LPR;
    const int ntasks = (int)(K / 256);
    const size_t rb = (size_t)ntasks * TB;
    warp_emu::run([&] {
        const int lane = (int)(threadIdx.x & 31);
        // the kernel's activation quantizer: one act-task per half-warp and round
        for (int i0 = 0; i0 < ntasks; i0 += 2) {
            const int t = i0 + (lane >> 4);
            const bool ok = t < ntasks;
            sb_quantize_task_h<true>(x, ok, rec, ok ? t : 0);
        }
        pthread_barrier_wait(&warp_emu::barrier());
        // activation-stationary: this lane's half act-task into registers once, then two rows per pass
        q45_acts A;
        if ((lane >> 1) < ntasks) q45_load_acts(rec, lane >> 1, lane & 1, A);
        rows_regs<T, 2>(rows, nrows, rb, A, lane, ntasks, out_regs, out_lanes);
        // task per lane (LPR = 16): half-warp `sub` takes the odd / even rows, the row sum by xor 8, 4, 2, 1
        const int sub = lane / LPR, l = lane % LPR;
        for (int r0 = 0; r0 < nrows; r0 += 32 / LPR) {
            const int r = r0 + sub;
            float acc = 0.0f;
            if (r < nrows)
                for (int t = l; t < ntasks; t += LPR) acc += task_dot<T>(rows + (size_t)r * rb + (size_t)t * TB, rec, t);
            for (int o = LPR / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (l == 0 && r < nrows) out_tasks[r] = acc;
        }
    });
}

extern "C" {

// x: K activations, quantized in the emulated warp into rec (K / 256 records of SB_REC bytes); rows: nrows packed rows.
// out_regs[nrows]: the activation-stationary results (the storing lane's); out_lanes[nrows][32]: the value of every lane that holds row r
// (lanes 0 .. 15 of its half-warp, the rest 0); out_tasks[nrows]: the task-per-lane results
int emu_sb_areg_rows(int type, const uint8_t * rows, int nrows, int64_t K, const float * x, uint8_t * rec, float * out_regs, float * out_lanes, float * out_tasks) {
    if (K % 256 != 0 || K < 256 || K > 16 * 256) return -1;
    if (type == T_Q4_K)      rows_both<T_Q4_K>(rows, nrows, K, x, rec, out_regs, out_lanes, out_tasks);
    else if (type == T_Q5_K) rows_both<T_Q5_K>(rows, nrows, K, x, rec, out_regs, out_lanes, out_tasks);
    else return -1;
    return 0;
}

int emu_sb_rec_bytes() { return SB_REC; }

} // extern "C"
