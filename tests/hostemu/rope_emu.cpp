// rope_emu.cpp — TEST INFRASTRUCTURE ONLY: ggml_b200/csrc/b200_rope.cuh (the per-pair math of the ROPE kernel) compiled for the host
// through tests/hostemu/shim and driven the way ops.cu's rope_kernel drives it (per position: the cos/sin cache, then every item of
// every row), exported with a C ABI for tests/test_hostemu_rope.py.  Catches pair-index, section and tail mistakes without a device.
#define B200_HOST_EMU 1
#include "cuda_shim.h"
#include <vector>
#include "../../ggml_b200/csrc/b200_rope.cuh"

using namespace b200;

template <typename T> static float ld(const uint8_t * p) {
    if constexpr (sizeof(T) == 4) return *(const float *)p; else return __half2float(*(const __half *)p);
}
template <typename T> static void st(uint8_t * p, float v) {
    if constexpr (sizeof(T) == 4) *(float *)p = v; else *(__half *)p = __float2half_rn(v);
}

template <typename T> static void rope_host(const int64_t * ne, const uint8_t * src, const size_t * snb, uint8_t * dst, const size_t * dnb,
                                            const int32_t * pos, const float * ff, const rope_consts & c) {
    std::vector<float> cs(ROPE_MAX_CACHE), sn(ROPE_MAX_CACHE);
    const int ncache = rope_n_cache(c);
    for (int64_t i3 = 0; i3 < ne[3]; ++i3)
        for (int64_t i2 = 0; i2 < ne[2]; ++i2) {
            float p[4] = { (float)pos[i2], 0.0f, 0.0f, 0.0f };
            if (c.mode & ROPE_MROPE) { p[1] = (float)pos[i2 + ne[2]]; p[2] = (float)pos[i2 + 2 * ne[2]]; p[3] = (float)pos[i2 + 3 * ne[2]]; }
            for (int j = 0; j < ncache; ++j) rope_cos_sin(c, rope_theta(c, p, j), ff ? ff[j] : 1.0f, j, cs[j], sn[j]);
            for (int64_t i1 = 0; i1 < ne[1]; ++i1) {
                const uint8_t * sr = src + i1 * snb[1] + i2 * snb[2] + i3 * snb[3];
                uint8_t * dr = dst + i1 * dnb[1] + i2 * dnb[2] + i3 * dnb[3];
                for (int64_t q = 0; q < ne[0] / 2; ++q) {
                    int64_t e0, e1;
                    const int slot = rope_item(c, q, e0, e1);
                    if (slot < 0) {
                        std::memcpy(dr + e0 * sizeof(T), sr + e0 * sizeof(T), sizeof(T));
                        std::memcpy(dr + e1 * sizeof(T), sr + e1 * sizeof(T), sizeof(T));
                        continue;
                    }
                    float y0, y1;
                    rope_rotate(ld<T>(sr + e0 * sizeof(T)), ld<T>(sr + e1 * sizeof(T)), cs[slot], sn[slot], y0, y1);
                    st<T>(dr + e0 * sizeof(T), y0); st<T>(dr + e1 * sizeof(T), y1);
                }
            }
        }
}

extern "C" {

// type 0 f32, 1 f16; ne / snb / dnb as ggml (elements / bytes); params laid out as ggml_b200_rope_params (include/ggml-b200.h)
int emu_rope(int type, const int64_t * ne, const uint8_t * src, const size_t * snb, uint8_t * dst, const size_t * dnb, const int32_t * pos,
             const float * ff, const rope_consts * params) {
    if (rope_n_cache(*params) > ROPE_MAX_CACHE) return -1;
    if (type == 0) rope_host<float>(ne, src, snb, dst, dnb, pos, ff, *params);
    else if (type == 1) rope_host<__half>(ne, src, snb, dst, dnb, pos, ff, *params);
    else return -1;
    return 0;
}

} // extern "C"
