// conv_emu.cpp — TEST INFRASTRUCTURE ONLY: ggml_b200/csrc/b200_conv.cuh (the per-element logic of IM2COL) compiled for the host through
// tests/hostemu/shim and driven the way ops.cu's im2col_kernel drives it (one output element at a time, in dst's order, rounded to fp16 by
// __float2half_rn for an f16 dst), exported with a C ABI for tests/test_hostemu_im2col.py.
#define B200_HOST_EMU 1
#include "cuda_shim.h"
#include "../../ggml_b200/csrc/b200_conv.cuh"
#include "check_code.h"

using namespace b200;

extern "C" {

// dst (packed, f32 or f16 per dst->type) = IM2COL(src0, src1) with the launcher's arguments; returns check_im2col's code and writes
// nothing unless it is 0
int emu_im2col(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, const ggml_b200_im2col_params * params) {
    const op_check r = check_im2col(src0, src1, dst, params);
    if (!r.ok()) return code(r);
    const im2col_geom g = im2col_geometry(*src0, *src1, *dst, *params);
    const int64_t n = nelem(*dst);
    for (int64_t e = 0; e < n; ++e) {
        const float v = im2col_value(g, (const uint8_t *)src1->data, e);
        if (dst->type == GGML_B200_TYPE_F32) ((float *)dst->data)[e] = v;
        else ((__half *)dst->data)[e] = __float2half_rn(v);
    }
    return 0;
}

} // extern "C"
