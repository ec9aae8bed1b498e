// wkv_emu.cpp — TEST INFRASTRUCTURE ONLY: ggml_b200/csrc/b200_wkv.cuh (the per-element math of RWKV_WKV6 and GATED_LINEAR_ATTN) compiled
// for the host through tests/hostemu/shim and driven the way ops.cu's wkv_kernel drives it (per sequence, head and column, the sequence's
// tokens in order, q * scale rounded once per token and row), exported with a C ABI for tests/test_hostemu_wkv.py.
#define B200_HOST_EMU 1
#include "cuda_shim.h"
#include "../../ggml_b200/csrc/b200_wkv.cuh"

#include <vector>

using namespace b200;

namespace {

// a = r (WKV6) or q (GLA), b = td or g; all packed as the C ABI requires; dst: y [S H, T], then the final states
void emu_wkv(bool gla, const float * k, const float * v, const float * a, const float * tf, const float * b, const float * s0, float * dst,
             int64_t S, int64_t H, int64_t T, int64_t n_seqs, float scale) {
    const int64_t C = S * H, n_seq_tok = T / n_seqs;
    std::vector<float> qs((size_t)S);
    for (int64_t s = 0; s < n_seqs; ++s)
        for (int64_t h = 0; h < H; ++h) {
            const int64_t head_state = (s * H + h) * S * S;
            float * st = dst + T * C + head_state;
            for (int64_t t = s * n_seq_tok; t < (s + 1) * n_seq_tok; ++t) {
                const int64_t base = t * C + h * S;
                const float * prev = t == s * n_seq_tok ? s0 + head_state : st;
                if (gla) for (int64_t i = 0; i < S; ++i) qs[(size_t)i] = gla_scaled_q(a[base + i], scale);
                for (int64_t j = 0; j < S; ++j)
                    dst[base + j] = gla ? gla_column(k + base, qs.data(), b + base, v[base + j], prev + j, st + j, S, S)
                                        : wkv6_column(k + base, a + base, tf + h * S, b + base, v[base + j], prev + j, st + j, S, S);
            }
        }
}

} // namespace

extern "C" {

void emu_rwkv_wkv6(const float * k, const float * v, const float * r, const float * tf, const float * td, const float * s0, float * dst,
                   int64_t S, int64_t H, int64_t T, int64_t n_seqs) {
    emu_wkv(false, k, v, r, tf, td, s0, dst, S, H, T, n_seqs, 1.0f);
}

void emu_gated_linear_attn(const float * k, const float * v, const float * q, const float * g, const float * s0, float * dst,
                           int64_t S, int64_t H, int64_t T, int64_t n_seqs, float scale) {
    emu_wkv(true, k, v, q, nullptr, g, s0, dst, S, H, T, n_seqs, scale);
}

} // extern "C"
