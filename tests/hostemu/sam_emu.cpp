// sam_emu.cpp — TEST INFRASTRUCTURE ONLY: ggml_b200/csrc/b200_sam.cuh (the per-row / per-element logic of WIN_PART, WIN_UNPART, GET_REL_POS,
// ADD_REL_POS and CONV_TRANSPOSE_2D) compiled for the host through tests/hostemu/shim and driven the way ops.cu's kernels drive it (one dst row
// or element at a time, with the launchers' arguments), plus the five checks of b200_op_checks.h, exported with a C ABI for
// tests/test_hostemu_sam.py.
#define B200_HOST_EMU 1
#include "cuda_shim.h"
#include "../../ggml_b200/csrc/b200_sam.cuh"
#include "../../ggml_b200/csrc/b200_op_checks.h"

#include <cstring>

using namespace b200;

namespace {
int code(const op_check & r) { return r.ok() || r.reason ? r.code : 1; }       // 1: a refusal without a reason
}

extern "C" {

// Each emu_X computes dst = X(src) with the launcher's arguments and returns check_X's code; it writes nothing unless that is 0.
int emu_win_part(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t npx, int32_t npy, int32_t w) {
    const op_check r = check_win_part(src, dst, npx, npy, w);
    if (!r.ok()) return code(r);
    const win_geom g{ w, npx, (int32_t)src->ne[1], (int32_t)src->ne[2] };
    const int64_t ne0 = dst->ne[0], rows = nrows(*dst);
    const uint32_t * s = (const uint32_t *)src->data;
    uint32_t * d = (uint32_t *)dst->data;
    for (int64_t row = 0; row < rows; ++row) {
        const int32_t sr = win_part_src_row(g, (uint32_t)row);
        for (int64_t i0 = 0; i0 < ne0; ++i0) d[row * ne0 + i0] = sr < 0 ? 0u : s[(int64_t)sr * ne0 + i0];
    }
    return 0;
}

int emu_win_unpart(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t w) {
    const op_check r = check_win_unpart(src, dst, w);
    if (!r.ok()) return code(r);
    const win_geom g{ w, (int32_t)((dst->ne[1] + w - 1) / w), (int32_t)dst->ne[1], (int32_t)dst->ne[2] };
    const int64_t ne0 = dst->ne[0], rows = nrows(*dst);
    const uint32_t * s = (const uint32_t *)src->data;
    uint32_t * d = (uint32_t *)dst->data;
    for (int64_t row = 0; row < rows; ++row)
        for (int64_t i0 = 0; i0 < ne0; ++i0) d[row * ne0 + i0] = s[(int64_t)win_unpart_src_row(g, (uint32_t)row) * ne0 + i0];
    return 0;
}

int emu_get_rel_pos(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    const op_check r = check_get_rel_pos(src, dst);
    if (!r.ok()) return code(r);
    const int64_t ne0 = dst->ne[0], rows = nrows(*dst);
    const uint16_t * s = (const uint16_t *)src->data;
    uint16_t * d = (uint16_t *)dst->data;
    for (int64_t row = 0; row < rows; ++row)
        for (int64_t i0 = 0; i0 < ne0; ++i0) d[row * ne0 + i0] = s[(int64_t)get_rel_pos_src_row((uint32_t)dst->ne[1], (uint32_t)row) * ne0 + i0];
    return 0;
}

// in place when dst->data == src0->data, as the kernel: each element is read before it is written
int emu_add_rel_pos(const ggml_b200_tensor * src0, const ggml_b200_tensor * pw, const ggml_b200_tensor * ph, const ggml_b200_tensor * dst) {
    const op_check r = check_add_rel_pos(src0, pw, ph, dst);
    if (!r.ok()) return code(r);
    const uint32_t L = (uint32_t)pw->ne[0], LL = (uint32_t)dst->ne[0];
    const int64_t rows = nrows(*dst);
    const float * s = (const float *)src0->data, * w = (const float *)pw->data, * h = (const float *)ph->data;
    float * d = (float *)dst->data;
    for (int64_t row = 0; row < rows; ++row)
        for (uint32_t c = 0; c < LL; ++c) {
            const uint32_t kh = c / L, kw = c - kh * L;
            d[row * LL + c] = add_rel_pos_value(s[row * LL + c], w[row * L + kw], h[row * L + kh], kh, kw);
        }
    return 0;
}

int emu_conv_transpose_2d(const ggml_b200_tensor * kernel, const ggml_b200_tensor * input, const ggml_b200_tensor * dst, int32_t stride) {
    const op_check r = check_conv_transpose_2d(kernel, input, dst, stride);
    if (!r.ok()) return code(r);
    const ct2d_geom g = ct2d_geometry(*kernel, *input, *dst, stride);
    float * d = (float *)dst->data;
    for (int32_t co = 0; co < g.Cout; ++co)
        for (int32_t oy = 0; oy < g.OH; ++oy)
            for (int32_t ox = 0; ox < g.OW; ++ox)
                d[((int64_t)co * g.OH + oy) * g.OW + ox] = ct2d_value(g, (const uint8_t *)kernel->data, (const uint8_t *)input->data, ox, oy, co);
    return 0;
}

// the checks alone (no data is touched)
int emu_check_win_part(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t npx, int32_t npy, int32_t w) { return code(check_win_part(src, dst, npx, npy, w)); }
int emu_check_win_unpart(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t w) { return code(check_win_unpart(src, dst, w)); }
int emu_check_get_rel_pos(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) { return code(check_get_rel_pos(src, dst)); }
int emu_check_add_rel_pos(const ggml_b200_tensor * src0, const ggml_b200_tensor * pw, const ggml_b200_tensor * ph, const ggml_b200_tensor * dst) {
    return code(check_add_rel_pos(src0, pw, ph, dst));
}
int emu_check_conv_transpose_2d(const ggml_b200_tensor * kernel, const ggml_b200_tensor * input, const ggml_b200_tensor * dst, int32_t stride) {
    return code(check_conv_transpose_2d(kernel, input, dst, stride));
}

} // extern "C"
