// pool_emu.cpp — TEST INFRASTRUCTURE ONLY: ggml_b200/csrc/b200_pool.cuh (the per-element logic of POOL_2D, UPSCALE, LEAKY_RELU and REPEAT)
// compiled for the host through tests/hostemu/shim and driven the way ops.cu's pool2d_kernel / upscale_kernel / leaky_relu_kernel /
// repeat_kernel drive it (one dst element at a time, in dst's order, with the launchers' arguments), plus the four checks of
// b200_op_checks.h, exported with a C ABI for tests/test_hostemu_pool.py.
#define B200_HOST_EMU 1
#include "cuda_shim.h"
#include "../../ggml_b200/csrc/b200_pool.cuh"
#include "../../ggml_b200/csrc/b200_op_checks.h"

#include <cstring>

using namespace b200;

namespace {
int code(const op_check & r) { return r.ok() || r.reason ? r.code : 1; }       // 1: a refusal without a reason
}

extern "C" {

// Each emu_X computes dst = X(src) with the launcher's arguments and returns check_X's code; it writes nothing unless that is 0.
int emu_pool_2d(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, const ggml_b200_pool_params * params) {
    const op_check r = check_pool_2d(src, dst, params);
    if (!r.ok()) return code(r);
    const pool2d_geom g = pool2d_geometry(*src, *dst, *params);
    const int64_t n = nelem(*dst);
    for (int64_t e = 0; e < n; ++e) ((float *)dst->data)[e] = pool2d_value(g, (const uint8_t *)src->data, e);
    return 0;
}

int emu_upscale(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    const op_check r = check_upscale(src, dst);
    if (!r.ok()) return code(r);
    const upscale_geom g = upscale_geometry(*src, *dst);
    const int64_t n = nelem(*dst);
    for (int64_t e = 0; e < n; ++e) {
        int64_t dofs;
        const int64_t sofs = upscale_offsets(g, e, dofs);
        memcpy((uint8_t *)dst->data + dofs, (const uint8_t *)src->data + sofs, 4);
    }
    return 0;
}

int emu_leaky_relu(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, float slope) {
    const op_check r = check_leaky_relu(src, dst);
    if (!r.ok()) return code(r);
    const ggml_b200_tensor & s = *src, & d = *dst;
    const int64_t n = nelem(d);
    for (int64_t e = 0; e < n; ++e) {
        const int64_t i0 = e % d.ne[0], i1 = (e / d.ne[0]) % d.ne[1], i2 = (e / (d.ne[0] * d.ne[1])) % d.ne[2], i3 = e / (d.ne[0] * d.ne[1] * d.ne[2]);
        const float x = *(const float *)((const uint8_t *)s.data + i0 * 4 + i1 * s.nb[1] + i2 * s.nb[2] + i3 * s.nb[3]);
        *(float *)((uint8_t *)d.data + i0 * 4 + i1 * d.nb[1] + i2 * d.nb[2] + i3 * d.nb[3]) = leaky_relu_value(x, slope);
    }
    return 0;
}

int emu_repeat(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    const op_check r = check_repeat(src, dst);
    if (!r.ok()) return code(r);
    const repeat_geom g = repeat_geometry(*src, *dst);
    const size_t es = repeat_elem_size(src->type);
    const int64_t n = nelem(*dst);
    for (int64_t e = 0; e < n; ++e) {
        int64_t dofs;
        const int64_t sofs = repeat_offsets(g, e, dofs);
        memcpy((uint8_t *)dst->data + dofs, (const uint8_t *)src->data + sofs, es);
    }
    return 0;
}

// the checks alone (no data is touched)
int emu_check_pool_2d(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, const ggml_b200_pool_params * params) { return code(check_pool_2d(src, dst, params)); }
int emu_check_upscale(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) { return code(check_upscale(src, dst)); }
int emu_check_leaky_relu(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) { return code(check_leaky_relu(src, dst)); }
int emu_check_repeat(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) { return code(check_repeat(src, dst)); }

} // extern "C"
