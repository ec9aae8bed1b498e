// ssm_emu.cpp — TEST INFRASTRUCTURE ONLY: ggml_b200/csrc/b200_ssm.cuh (the per-element math of SSM_CONV and SSM_SCAN) compiled for the
// host through tests/hostemu/shim and driven the way ops.cu's ssm_conv_kernel / ssm_scan_kernel drive it (the same index and stride
// arithmetic per output element, resp. per row and sequence over the tokens), exported with a C ABI for tests/test_hostemu_ssm.py.
#define B200_HOST_EMU 1
#include "cuda_shim.h"
#include "../../ggml_b200/csrc/b200_ssm.cuh"

using namespace b200;

extern "C" {

struct emu_tensor { const uint8_t * data; int64_t ne[4]; uint64_t nb[4]; };    // a source as the kernels see it (ne, byte strides)

// dst f32 [d_inner, n_t, n_s], contiguous = SSM_CONV(sx, c)
void emu_ssm_conv(const emu_tensor * sx, const emu_tensor * c, float * dst, int64_t n_t) {
    const int64_t d_inner = sx->ne[1], n_s = sx->ne[2];
    for (int64_t s = 0; s < n_s; ++s)
        for (int64_t t = 0; t < n_t; ++t)
            for (int64_t i1 = 0; i1 < d_inner; ++i1) {
                const float * win = (const float *)(sx->data + i1 * sx->nb[1] + s * sx->nb[2]) + t;
                const float * w = (const float *)(c->data + i1 * c->nb[1]);
                dst[(s * n_t + t) * d_inner + i1] = ssm_conv_dot(win, w, c->ne[0]);
            }
}

// dst f32, contiguous: y [d_inner, n_t, n_s], then the final states [d_state, d_inner, n_s] = SSM_SCAN(t[0..5] = s, x, dt, A, B, C);
// s, x, dt, A contiguous (as the C ABI requires), B and C any nb1 / nb2
void emu_ssm_scan(const emu_tensor * t, float * dst) {
    const emu_tensor & s0 = t[0], & x = t[1], & dt = t[2], & A = t[3], & B = t[4], & C = t[5];
    const int64_t nc = s0.ne[0], d_inner = s0.ne[1], n_s = s0.ne[2], n_t = x.ne[1];
    uint8_t * d = (uint8_t *)dst;
    for (int64_t s = 0; s < n_s; ++s)
        for (int64_t i1 = 0; i1 < d_inner; ++i1) {
            const float * a = (const float *)(A.data + i1 * A.nb[1]);
            const float * prev = (const float *)(s0.data + i1 * s0.nb[1] + s * s0.nb[2]);
            float * st = (float *)(d + x.nb[3] + i1 * s0.nb[1] + s * s0.nb[2]);
            for (int64_t k = 0; k < n_t; ++k) {
                const float xv = *(const float *)(x.data + i1 * x.nb[0] + k * x.nb[1] + s * x.nb[2]);
                const float dv = *(const float *)(dt.data + i1 * dt.nb[0] + k * dt.nb[1] + s * dt.nb[2]);
                const float * b = (const float *)(B.data + k * B.nb[1] + s * B.nb[2]);
                const float * cc = (const float *)(C.data + k * C.nb[1] + s * C.nb[2]);
                *(float *)(d + i1 * x.nb[0] + k * x.nb[1] + s * x.nb[2]) = ssm_scan_token(prev, st, a, b, cc, xv, dv, nc);
                prev = st;
            }
        }
}

} // extern "C"
