// b200_sort.cuh — the row sort of GGML_OP_ARGSORT: a bitonic network over (key, index) pairs, one row of at most SORT_MAX_COLS values.
// __host__ __device__, so that tests/hostemu compiles the same compare-exchange steps for the CPU and runs them in the device's order.
//
// Each element becomes one 64-bit item, key << 32 | index, and the network sorts the items ascending.  The key maps the float to an
// unsigned integer whose order is the requested order, so the items are unique and their order is a strict total order:
//   * -0.0 and +0.0 get the same key (they compare equal, as in ggml-cpu);
//   * equal keys are ordered by the index in the low half: ties come out in ascending source index, in both orders;
//   * every NaN (any sign or payload) gets the largest key, 0xFFFFFFFF, in both orders: NaNs sort after every number;
//   * the padding up to the next power of two is (0xFFFFFFFF, index >= ne0): after the NaNs, so the first ne0 items hold exactly the
//     indices 0 .. ne0-1.
// The low 32 bits of the first ne0 sorted items are the result: always a permutation of 0 .. ne0-1, whatever the values.
#pragma once

#include <cstdint>
#include <cstring>

#include "b200_op_checks.h"     // SORT_MAX_COLS, SORT_ASC / SORT_DESC

namespace b200 {

__host__ __device__ __forceinline__ uint32_t sort_key(float v, int order) {
    if (v != v) return 0xFFFFFFFFu;                                   // NaN: last in both orders
    if (v == 0.0f) v = 0.0f;                                          // -0.0 -> +0.0
    uint32_t u;
#ifdef __CUDA_ARCH__
    u = __float_as_uint(v);
#else
    std::memcpy(&u, &v, sizeof(u));
#endif
    const uint32_t asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // monotone: -inf -> 0x007FFFFF ... +inf -> 0xFF800000
    return order == SORT_DESC ? ~asc : asc;                           // both stay in [0x007FFFFF, 0xFF800000], below the NaN key
}

// item i of a row of ne0 values (i < ne0: the value x; otherwise padding)
__host__ __device__ __forceinline__ uint64_t sort_item(float x, int32_t i, int order) {
    return ((uint64_t)sort_key(x, order) << 32) | (uint32_t)i;
}
__host__ __device__ __forceinline__ uint64_t sort_pad(int32_t i) { return (0xFFFFFFFFull << 32) | (uint32_t)i; }

// the padded row length: the next power of two >= ne0 (ne0 >= 1)
__host__ __device__ __forceinline__ int sort_width(int ne0) {
    int p = 1;
    while (p < ne0) p <<= 1;
    return p;
}

// one compare-exchange of the bitonic network over s[0 .. P): stage k (2, 4, .. P), distance j (k/2, k/4, .. 1), pair t (0 .. P/2).
// The P/2 pairs of one (k, j) step are disjoint, so they may run in any order or all at once; the steps run in sequence.
__host__ __device__ __forceinline__ void sort_step(uint64_t * s, int k, int j, int t) {
    const int i = 2 * j * (t / j) + (t % j), l = i + j;
    const bool up = (i & k) == 0;
    const uint64_t a = s[i], b = s[l];
    if ((a > b) == up) { s[i] = b; s[l] = a; }
}

} // namespace b200
