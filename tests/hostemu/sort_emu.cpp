// sort_emu.cpp — TEST INFRASTRUCTURE ONLY: ggml_b200/csrc/b200_sort.cuh (the ARGSORT network) compiled for the host through
// tests/hostemu/shim and driven the way ops.cu's argsort_kernel drives it (per row: the padded items, then every (k, j) step over all
// pairs), exported with a C ABI for tests/test_hostemu_sort.py.
#define B200_HOST_EMU 1
#include "cuda_shim.h"
#include <vector>
#include "../../ggml_b200/csrc/b200_sort.cuh"

using namespace b200;

extern "C" {

// rows contiguous rows of ne0 f32 values -> rows x ne0 i32 indices; returns -1 outside 1 <= ne0 <= SORT_MAX_COLS
int emu_argsort(const float * x, int64_t ne0, int64_t rows, int order, int32_t * out) {
    if (ne0 < 1 || ne0 > SORT_MAX_COLS || (order != SORT_ASC && order != SORT_DESC)) return -1;
    const int P = sort_width((int)ne0);
    std::vector<uint64_t> items(P);
    for (int64_t r = 0; r < rows; ++r) {
        for (int i = 0; i < P; ++i) items[i] = i < ne0 ? sort_item(x[r * ne0 + i], i, order) : sort_pad(i);
        for (int k = 2; k <= P; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1)
                for (int t = 0; t < P / 2; ++t) sort_step(items.data(), k, j, t);
        for (int64_t i = 0; i < ne0; ++i) out[r * ne0 + i] = (int32_t)(uint32_t)items[i];
    }
    return 0;
}

} // extern "C"
