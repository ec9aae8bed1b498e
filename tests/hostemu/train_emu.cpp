// train_emu.cpp — TEST INFRASTRUCTURE ONLY: ggml_b200/csrc/b200_train.cuh (the per-element logic of OUT_PROD, OPT_STEP_ADAMW, ARGMAX,
// REPEAT_BACK, STEP and the cross-entropy pair) compiled for the host through tests/hostemu/shim and driven the way ops.cu's kernels drive it,
// exported with a C ABI for tests/test_hostemu_train.py.
#define B200_HOST_EMU 1
#include "cuda_shim.h"
#include "../../ggml_b200/csrc/b200_train.cuh"
#include "check_code.h"

using namespace b200;

extern "C" {

// w, m, v updated in place over n elements with params[7], as opt_step_adamw_kernel does
void emu_adamw(int64_t n, float * w, const float * g, float * m, float * v, const float * params) {
    for (int64_t i = 0; i < n; ++i) adamw_update(w[i], g[i], m[i], v[i], params);
}

int32_t emu_argmax_closed(const float * x, int64_t n) { return argmax_row_closed(x, n); }
int32_t emu_argmax_seq(const float * x, int64_t n) { return argmax_row_seq(x, n); }

// dst = OUT_PROD(src0, src1), each output the fused chain of out_prod_step in ascending k; returns check_out_prod's code
int emu_out_prod(const ggml_b200_tensor * a, const ggml_b200_tensor * b, const ggml_b200_tensor * d) {
    const op_check r = check_out_prod(a, b, d);
    if (!r.ok()) return code(r);
    const int64_t K = a->ne[1], dps2 = d->ne[2] / a->ne[2], dps3 = d->ne[3] / a->ne[3];
    for (int64_t i3 = 0; i3 < d->ne[3]; ++i3)
        for (int64_t i2 = 0; i2 < d->ne[2]; ++i2)
            for (int64_t i1 = 0; i1 < d->ne[1]; ++i1)
                for (int64_t i0 = 0; i0 < d->ne[0]; ++i0) {
                    float acc = 0.0f;
                    for (int64_t k = 0; k < K; ++k) {
                        const float x = *(const float *)((const uint8_t *)a->data + i0 * 4 + k * a->nb[1] + (i2 / dps2) * a->nb[2] + (i3 / dps3) * a->nb[3]);
                        const float y = *(const float *)((const uint8_t *)b->data + i1 * b->nb[0] + k * b->nb[1] + i2 * b->nb[2] + i3 * b->nb[3]);
                        acc = out_prod_step(acc, x, y);
                    }
                    *(float *)((uint8_t *)d->data + i0 * 4 + i1 * d->nb[1] + i2 * d->nb[2] + i3 * d->nb[3]) = acc;
                }
    return 0;
}

// dst = REPEAT_BACK(src) element by element, as repeat_back_kernel; returns check_repeat_back's code
int emu_repeat_back(const ggml_b200_tensor * s, const ggml_b200_tensor * d) {
    const op_check r = check_repeat_back(s, d);
    if (!r.ok()) return code(r);
    const repeat_back_geom g = repeat_back_geometry(*s, *d);
    const int64_t n = nelem(*d);
    for (int64_t e = 0; e < n; ++e) {
        float v;
        const int64_t off = repeat_back_value(g, (const uint8_t *)s->data, e, &v);
        *(float *)((uint8_t *)d->data + off) = v;
    }
    return 0;
}

void emu_step(const float * x, float * y, int64_t n) { for (int64_t i = 0; i < n; ++i) y[i] = step_value(x[i]); }

} // extern "C"
