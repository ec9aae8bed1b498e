// b200_op_checks.h — what each op launcher of ops.cu accepts, decided in one place.  Every ggml_b200_op_* below returns
// the verdict of its check before it launches anything, and the backend's supports_op asks the same check for each such node, on descriptors
// built by the same code that builds the launch's (bound_op in backend/ggml-b200.cpp), so that a node the plug-in accepts is one its
// launcher runs.  The checks read only the descriptors and the op's scalars: what the launcher cannot see (graph structure, ggml-cpu's
// own layout assumptions) stays with the caller.  Conditions that matter only for a launch (the grid limits) come after the empty-tensor
// early return, in the order the launchers have always applied them.
//
// Host-only C++: the ABI header and the standard library, no CUDA and no ggml headers, so the plug-in, the launchers and the CPU tests
// compile the same rules.
#pragma once

#include "../../include/ggml-b200.h"

#include <algorithm>
#include <cstdint>

namespace b200 {

enum { ROPE_NORM = 0, ROPE_NEOX = 2, ROPE_MROPE = 8, ROPE_VISION = 24 };
enum { ROPE_MAX_CACHE = 512 };              // cos/sin pairs per position held in shared memory: n_dims <= 1024
enum { SORT_MAX_COLS = 1024 };              // row length limit (ne0) of the one-CTA ARGSORT network: 1024 items, 8 KB of shared memory
enum { SORT_ASC = 0, SORT_DESC = 1 };       // enum ggml_sort_order
enum { WKV_COLS = 32 };                     // RWKV_WKV6 / GATED_LINEAR_ATTN: state columns per CTA (one warp, one column per lane)
enum { WKV_MAX_HEAD = 256 };                // their head size limit: S rows x WKV_COLS columns of state plus four S-vectors, 36 KB of shared memory

// the shared memory of one RWKV_WKV6 / GATED_LINEAR_ATTN CTA for head size S: the state block, then the token's k, r / q, td / g and tf
inline size_t wkv_smem_bytes(int64_t S) { return (size_t)S * (WKV_COLS + 4) * sizeof(float); }

// number of cos/sin entries a position needs: pairs j < n_dims/2, or j < n_dims (= ne0/2) in VISION mode
#ifdef __CUDACC__
__host__ __device__ __forceinline__
#else
inline
#endif
int rope_n_cache(const ggml_b200_rope_params & c) { return c.mode == ROPE_VISION ? c.n_dims : c.n_dims / 2; }

// the ROPE grid is (positions, blocks of heads, batches): a CTA takes as many whole heads as fit in 256 elements, at least one (ne0 > 0)
inline int rope_heads_per_cta(int64_t ne0) { return (int)std::max<int64_t>(1, 256 / ne0); }

struct op_check {
    int          code;     // GGML_B200_OK, or what the launcher returns: GGML_B200_EUNSUPPORTED or GGML_B200_EINVAL
    const char * reason;   // nullptr when accepted
    bool ok() const { return code == GGML_B200_OK; }
};
constexpr op_check accepted{ GGML_B200_OK, nullptr };

inline int64_t nelem(const ggml_b200_tensor & t) { return t.ne[0] * t.ne[1] * t.ne[2] * t.ne[3]; }
inline int64_t nrows(const ggml_b200_tensor & t) { return t.ne[1] * t.ne[2] * t.ne[3]; }
inline bool same_shape(const ggml_b200_tensor & a, const ggml_b200_tensor & b) {
    return a.ne[0] == b.ne[0] && a.ne[1] == b.ne[1] && a.ne[2] == b.ne[2] && a.ne[3] == b.ne[3];
}
inline bool is_float(int32_t t) { return t == GGML_B200_TYPE_F32 || t == GGML_B200_TYPE_F16; }
// a tensor of es-byte elements stored without gaps, in ggml's order
inline bool is_packed(const ggml_b200_tensor & t, size_t es) {
    size_t nb = es;
    for (int i = 0; i < 4; ++i) { if (t.ne[i] != 1 && t.nb[i] != nb) return false; nb *= (size_t)t.ne[i]; }
    return true;
}
inline bool is_packed4(const ggml_b200_tensor & t) { return is_packed(t, 4); }      // f32, i32

// the output extent of a convolution along one axis (ggml_calc_conv_output_size, src/ggml.c:3770)
inline int64_t conv_out_size(int64_t ins, int64_t ks, int64_t s, int64_t p, int64_t d) { return (ins + 2 * p - d * (ks - 1) - 1) / s + 1; }

// the block formats this library decodes (every one of them also runs the quantized MUL_MAT / MUL_MAT_ID)
inline bool is_block_type(int32_t t) {
    switch (t) {
        case GGML_B200_TYPE_Q4_0: case GGML_B200_TYPE_Q8_0: case GGML_B200_TYPE_Q4_K: case GGML_B200_TYPE_Q5_K: case GGML_B200_TYPE_Q6_K:
        case GGML_B200_TYPE_Q4_1: case GGML_B200_TYPE_Q5_0: case GGML_B200_TYPE_Q5_1: case GGML_B200_TYPE_Q2_K: case GGML_B200_TYPE_Q3_K:
        case GGML_B200_TYPE_IQ4_NL: case GGML_B200_TYPE_IQ4_XS:
        case GGML_B200_TYPE_IQ2_XXS: case GGML_B200_TYPE_IQ3_XXS: case GGML_B200_TYPE_IQ1_S:
        case GGML_B200_TYPE_IQ2_XS: case GGML_B200_TYPE_IQ2_S: case GGML_B200_TYPE_IQ3_S: case GGML_B200_TYPE_IQ1_M:
        case GGML_B200_TYPE_TQ1_0: case GGML_B200_TYPE_TQ2_0:
            return true;
        default: return false;
    }
}

#define B200_REQUIRE(cond, why) do { if (!(cond)) return op_check{ GGML_B200_EUNSUPPORTED, why }; } while (0)
#define B200_VALID(cond, why)   do { if (!(cond)) return op_check{ GGML_B200_EINVAL, why }; } while (0)

constexpr int32_t F32 = GGML_B200_TYPE_F32, F16 = GGML_B200_TYPE_F16, I32 = GGML_B200_TYPE_I32;

inline op_check check_get_rows(const ggml_b200_tensor * src0, const ggml_b200_tensor * ids, const ggml_b200_tensor * dst) {
    B200_REQUIRE(dst->type == F32 && ids->type == I32, "dst must be f32, ids i32");
    B200_REQUIRE(is_float(src0->type) || is_block_type(src0->type), "unsupported row type");
    B200_REQUIRE(dst->nb[0] == 4, "dst rows must be contiguous");
    return accepted;
}

inline op_check check_bin_bcast(int32_t op, const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src0->type == F32 && src1->type == F32 && dst->type == F32, "f32 only");
    if (nelem(*dst) == 0) return accepted;
    B200_VALID(op >= 0 && op <= 3, "bad op (0 add, 1 mul, 2 sub, 3 div)");
    return accepted;
}

// NORM / RMS_NORM: the kernel writes dst's rows with src's extents
inline op_check check_norm(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src->type == F32 && dst->type == F32 && src->nb[0] == 4 && dst->nb[0] == 4, "f32 rows contiguous along dim 0");
    B200_VALID(same_shape(*src, *dst), "src and dst shapes differ");
    return accepted;
}

// NORM / RMS_NORM -> MUL(gain) -> ADD(bias): the kernel writes the three dsts' rows with src's extents and reads gain[i] and bias[i] for
// every i < ne0 through these two pointers
inline op_check check_norm_affine(const ggml_b200_tensor * src, const ggml_b200_tensor * dst_norm, const float * gain, const ggml_b200_tensor * dst_mul,
                                  const float * bias, const ggml_b200_tensor * dst_add) {
    B200_REQUIRE(src->type == F32 && dst_norm->type == F32 && dst_mul->type == F32 && dst_add->type == F32, "f32 only");
    B200_REQUIRE(src->nb[0] == 4 && dst_norm->nb[0] == 4 && dst_mul->nb[0] == 4 && dst_add->nb[0] == 4 && gain && bias, "rows contiguous along dim 0");
    B200_VALID(same_shape(*src, *dst_norm) && same_shape(*src, *dst_mul) && same_shape(*src, *dst_add), "the dsts must have src's shape");
    return accepted;
}

// ... with gain and bias described, as the launcher takes them: packed f32 [ne0] (nb0 == 4, every other extent 1)
inline op_check check_norm_affine(const ggml_b200_tensor * src, const ggml_b200_tensor * dst_norm, const ggml_b200_tensor * gain,
                                  const ggml_b200_tensor * dst_mul, const ggml_b200_tensor * bias, const ggml_b200_tensor * dst_add) {
    B200_REQUIRE(gain && bias, "gain and bias are required");
    B200_REQUIRE(gain->type == F32 && bias->type == F32 && gain->nb[0] == 4 && bias->nb[0] == 4, "gain and bias must be f32, contiguous");
    const op_check rows = check_norm_affine(src, dst_norm, (const float *) gain->data, dst_mul, (const float *) bias->data, dst_add);
    if (!rows.ok()) return rows;
    const int64_t n = src->ne[0];
    B200_VALID(gain->ne[0] == n && nelem(*gain) == n && bias->ne[0] == n && nelem(*bias) == n, "gain and bias must be [ne0]");
    return accepted;
}

// SCALE, and with it DIAG_MASK_INF and the unary functions: one thread per element of packed f32 tensors
inline op_check check_scale(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src && dst, "src and dst are required");
    B200_REQUIRE(src->type == F32 && dst->type == F32, "src and dst must be f32");
    B200_REQUIRE(is_packed4(*src) && is_packed4(*dst), "src and dst must be packed");
    B200_VALID(same_shape(*src, *dst), "src and dst shapes differ");
    if (nelem(*dst) == 0) return accepted;
    B200_REQUIRE((nelem(*dst) + 255) / 256 <= 0x7fffffff, "too many elements for one grid");
    return accepted;
}

inline op_check check_diag_mask_inf(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) { return check_scale(src, dst); }

inline op_check check_unary(int32_t uop, const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_VALID(uop >= 0 && uop <= GGML_B200_UNARY_STEP, "bad unary op (0 .. 13, enum ggml_b200_unary)");
    return check_scale(src, dst);
}

// SOFT_MAX: src and dst packed f32 of one shape, one CTA per row; the kernel reads mask row i1 at i1 ne0 elements, so the mask is what
// ggml_soft_max_impl asserts: a packed f32 or f16 matrix [ne0, >= ne1]
inline op_check check_soft_max(const ggml_b200_tensor * src, const ggml_b200_tensor * mask, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src && dst, "src and dst are required");
    B200_REQUIRE(src->type == F32 && dst->type == F32, "src and dst must be f32");
    B200_REQUIRE(is_packed4(*src) && is_packed4(*dst), "src and dst must be packed");
    B200_VALID(same_shape(*src, *dst), "src and dst shapes differ");
    if (mask) {
        B200_REQUIRE(is_float(mask->type) && is_packed(*mask, mask->type == F32 ? 4 : 2), "mask must be packed f32 or f16");
        B200_VALID(mask->ne[2] == 1 && mask->ne[3] == 1 && mask->ne[0] == src->ne[0] && mask->ne[1] >= src->ne[1], "mask must be [ne0, >= ne1]");
    }
    if (nelem(*src) == 0) return accepted;
    B200_REQUIRE(nrows(*src) <= 0x7fffffff, "too many rows for one grid");
    return accepted;
}

inline op_check check_cpy(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_REQUIRE(nelem(*src) == nelem(*dst), "element counts differ");
    if (nelem(*src) == 0) return accepted;
    if (is_float(src->type) && is_float(dst->type)) return accepted;
    B200_REQUIRE(src->type == F32 && (dst->type == GGML_B200_TYPE_Q8_0 || dst->type == GGML_B200_TYPE_Q4_0), "unsupported type pair");
    B200_REQUIRE(src->nb[0] == 4 && src->ne[0] % 32 == 0 && dst->ne[0] % 32 == 0, "f32 -> q needs dim-0 contiguous rows of whole blocks");
    return accepted;
}

inline op_check check_cpy2(const ggml_b200_tensor * src_a, const ggml_b200_tensor * dst_a, const ggml_b200_tensor * src_b, const ggml_b200_tensor * dst_b) {
    const int64_t n = nelem(*src_a);
    B200_REQUIRE(n == nelem(*dst_a) && n == nelem(*src_b) && n == nelem(*dst_b), "element counts differ");
    B200_REQUIRE(is_float(src_a->type) && is_float(dst_a->type) && is_float(src_b->type) && is_float(dst_b->type), "float tensors only");
    return accepted;
}

inline op_check check_flash_attn_ext(const ggml_b200_tensor * q, const ggml_b200_tensor * k, const ggml_b200_tensor * v, const ggml_b200_tensor * mask,
                                     const ggml_b200_tensor * dst) {
    auto decodable = [](int32_t t) { return is_float(t) || is_block_type(t); };
    B200_REQUIRE(q->type == F32 && dst->type == F32 && q->nb[0] == 4 && dst->nb[0] == 4, "q and dst must be f32 rows");
    B200_REQUIRE(decodable(k->type) && decodable(v->type), "unsupported K / V type");
    B200_REQUIRE(q->ne[0] >= 1 && q->ne[0] <= 256 && k->ne[0] == q->ne[0] && v->ne[0] == q->ne[0] && v->ne[1] == k->ne[1], "head size must be <= 256 and agree");
    B200_REQUIRE(k->ne[2] > 0 && k->ne[3] > 0 && v->ne[2] > 0 && v->ne[3] > 0 && q->ne[2] % k->ne[2] == 0 && q->ne[3] % k->ne[3] == 0 &&
                 q->ne[2] % v->ne[2] == 0 && q->ne[3] % v->ne[3] == 0, "heads do not broadcast");
    B200_REQUIRE(!mask || (mask->type == F16 && mask->nb[0] == 2 && mask->ne[0] >= k->ne[1] && mask->ne[1] >= q->ne[1]), "mask must be f16 [n_kv, >= n_q]");
    if (q->ne[1] == 0 || q->ne[2] == 0 || q->ne[3] == 0) return accepted;
    B200_REQUIRE(q->ne[2] <= 65535 && q->ne[3] <= 65535, "too many heads / batches for one grid");
    return accepted;
}

inline op_check check_mul_mat_f(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst) {
    const ggml_b200_tensor & a = *src0, & b = *src1, & d = *dst;
    // an f16 src1 only with an f16 src0: the CPU backend's vec_dot type for f16 weights, used as is (any other pair it converts first)
    B200_REQUIRE(is_float(a.type) && (b.type == F32 || (b.type == F16 && a.type == F16)) && d.type == F32, "f32/f16 x f32 or f16 x f16 -> f32");
    B200_REQUIRE(a.ne[0] == b.ne[0] && d.ne[0] == a.ne[1] && d.ne[1] == b.ne[1] && d.ne[2] == b.ne[2] && d.ne[3] == b.ne[3], "shape mismatch");
    B200_REQUIRE(b.ne[2] % a.ne[2] == 0 && b.ne[3] % a.ne[3] == 0, "batch dims do not broadcast");
    return accepted;
}

inline op_check check_rope(const ggml_b200_tensor * src, const ggml_b200_tensor * pos, const ggml_b200_tensor * freq_factors, const ggml_b200_tensor * dst,
                           const ggml_b200_rope_params * params) {
    B200_REQUIRE(src && pos && dst && params, "src, pos, dst and params are required");
    const ggml_b200_tensor & s = *src, & p = *pos, & d = *dst;
    const ggml_b200_rope_params & c = *params;
    B200_REQUIRE(is_float(s.type) && d.type == s.type, "src and dst must both be f32 or both f16");
    const size_t es = s.type == F32 ? 4 : 2;
    B200_REQUIRE(s.nb[0] == es && d.nb[0] == es, "rows must be contiguous along dim 0");
    B200_REQUIRE(same_shape(s, d), "src and dst shapes differ");
    B200_REQUIRE(c.mode == ROPE_NORM || c.mode == ROPE_NEOX || c.mode == ROPE_MROPE || c.mode == ROPE_VISION, "mode must be 0, 2, 8 or 24");
    B200_REQUIRE(c.n_dims >= 0 && c.n_dims % 2 == 0 && c.n_dims <= s.ne[0] && s.ne[0] % 2 == 0, "n_dims must be even and <= ne0 (ne0 even)");
    B200_REQUIRE(c.mode != ROPE_VISION || 2 * (int64_t)c.n_dims == s.ne[0], "VISION mode needs n_dims == ne0/2");
    if (c.mode & ROPE_MROPE) {
        B200_REQUIRE(c.sections[0] >= 0 && c.sections[1] >= 0 && c.sections[2] >= 0 && c.sections[3] >= 0, "sections must be >= 0");
        B200_REQUIRE(c.sections[0] > 0 || c.sections[1] > 0 || c.sections[2] > 0, "MROPE sections must not all be zero");
        B200_REQUIRE((int64_t)c.sections[0] + c.sections[1] + c.sections[2] + c.sections[3] <= s.ne[0], "MROPE sections exceed ne0");
    }
    const int ncache = rope_n_cache(c);
    B200_REQUIRE(ncache <= ROPE_MAX_CACHE, "n_dims too large (at most 1024 rotated dimensions)");
    B200_REQUIRE(p.type == I32 && p.nb[0] == 4 && p.ne[0] >= s.ne[2] * ((c.mode & ROPE_MROPE) ? 4 : 1), "pos must be i32, contiguous, one per position (four in MROPE)");
    if (freq_factors)
        B200_REQUIRE(freq_factors->type == F32 && freq_factors->nb[0] == 4 && freq_factors->ne[0] >= ncache,
                     "freq_factors must be f32, contiguous, >= n_dims/2 entries (n_dims in VISION mode)");
    if (s.ne[0] == 0 || s.ne[1] == 0 || s.ne[2] == 0 || s.ne[3] == 0) return accepted;
    const int hpc = rope_heads_per_cta(s.ne[0]);
    B200_REQUIRE(s.ne[2] <= 0x7fffffff && (s.ne[1] + hpc - 1) / hpc <= 65535 && s.ne[3] <= 65535, "too many positions / heads / batches for one grid");
    return accepted;
}

inline op_check check_argsort(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t order) {
    B200_REQUIRE(src && dst, "src and dst are required");
    B200_VALID(order == SORT_ASC || order == SORT_DESC, "bad order (0 ascending, 1 descending)");
    B200_REQUIRE(src->type == F32 && dst->type == I32, "src must be f32, dst i32");
    B200_REQUIRE(src->nb[0] == 4, "src rows must be contiguous along dim 0");
    B200_REQUIRE(same_shape(*src, *dst), "src and dst shapes differ");
    B200_REQUIRE(is_packed4(*dst), "dst must be contiguous");
    B200_REQUIRE(src->ne[0] <= SORT_MAX_COLS, "rows longer than 1024 are not supported");
    if (nrows(*src) == 0 || src->ne[0] == 0) return accepted;
    B200_REQUIRE(nrows(*src) <= 0x7fffffff, "too many rows for one grid");
    return accepted;
}

inline op_check check_sum_rows(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src && dst, "src and dst are required");
    const ggml_b200_tensor & s = *src, & d = *dst;
    B200_REQUIRE(s.type == F32 && d.type == F32, "src and dst must be f32");
    B200_REQUIRE(s.nb[0] == 4 && d.nb[0] == 4, "rows must be contiguous along dim 0");
    B200_REQUIRE(d.ne[0] == 1 && s.ne[1] == d.ne[1] && s.ne[2] == d.ne[2] && s.ne[3] == d.ne[3], "dst must be [1, ne1, ne2, ne3] of src");
    if (nrows(s) == 0) return accepted;
    B200_REQUIRE((nrows(s) + 3) / 4 <= 0x7fffffff, "too many rows for one grid");
    return accepted;
}

inline op_check check_concat(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, int32_t dim) {
    B200_REQUIRE(src0 && src1 && dst, "src0, src1 and dst are required");
    B200_VALID(dim >= 0 && dim <= 3, "bad dim (0 .. 3)");
    const ggml_b200_tensor & a = *src0, & b = *src1, & d = *dst;
    B200_REQUIRE((a.type == F32 || a.type == I32) && b.type == a.type && d.type == a.type, "src0, src1 and dst must all be f32 or all i32");
    B200_REQUIRE(a.nb[0] == 4, "src0 must be contiguous along dim 0");
    for (int k = 0; k < 4; ++k) {
        if (k == dim) B200_REQUIRE(d.ne[k] == a.ne[k] + b.ne[k], "dst's extent along dim must be src0's plus src1's");
        else B200_REQUIRE(a.ne[k] == b.ne[k] && d.ne[k] == a.ne[k], "src0, src1 and dst must agree outside dim");
    }
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE((nelem(d) + 255) / 256 <= 0x7fffffff, "too many elements for one grid");
    return accepted;
}

inline op_check check_ssm_conv(const ggml_b200_tensor * sx, const ggml_b200_tensor * c, const ggml_b200_tensor * dst) {
    B200_REQUIRE(sx && c && dst, "sx, c and dst are required");
    const ggml_b200_tensor & x = *sx, & w = *c, & d = *dst;
    B200_REQUIRE(x.type == F32 && w.type == F32 && d.type == F32, "sx, c and dst must be f32");
    B200_REQUIRE(x.nb[0] == 4 && w.nb[0] == 4 && d.nb[0] == 4, "sx, c and dst must be contiguous along dim 0");
    // ggml-cpu reads row i1 of sx at i1 * ne0 (it asserts so) and row i1 of c at i1 * d_conv (whatever c's nb1: only packed rows mean the
    // same data on both backends)
    B200_REQUIRE(x.nb[1] == (size_t)x.ne[0] * 4 && w.nb[1] == (size_t)w.ne[0] * 4, "the rows of sx and of c must be packed (nb1 == ne0 * 4)");
    B200_REQUIRE(x.ne[3] == 1 && w.ne[2] == 1 && w.ne[3] == 1, "sx must be 3-D and c a matrix");
    B200_REQUIRE(w.ne[1] == x.ne[1] && x.ne[0] - w.ne[0] + 1 >= 0, "c must be [d_conv, d_inner] with d_conv <= ne0 of sx + 1");
    B200_REQUIRE(d.ne[0] == x.ne[1] && d.ne[1] == x.ne[0] - w.ne[0] + 1 && d.ne[2] == x.ne[2] && d.ne[3] == 1, "dst must be [d_inner, n_t, n_s]");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE((nelem(d) + 255) / 256 <= 0x7fffffff, "too many elements for one grid");
    return accepted;
}

inline op_check check_ssm_scan(const ggml_b200_tensor * s, const ggml_b200_tensor * x, const ggml_b200_tensor * dt, const ggml_b200_tensor * A,
                               const ggml_b200_tensor * B, const ggml_b200_tensor * C, const ggml_b200_tensor * dst) {
    B200_REQUIRE(s && x && dt && A && B && C && dst, "s, x, dt, A, B, C and dst are required");
    const ggml_b200_tensor & ts = *s, & tx = *x, & tdt = *dt, & ta = *A, & tb = *B, & tc = *C, & d = *dst;
    B200_REQUIRE(ts.type == F32 && tx.type == F32 && tdt.type == F32 && ta.type == F32 && tb.type == F32 && tc.type == F32 && d.type == F32,
                 "all tensors must be f32");
    B200_REQUIRE(is_packed4(ts) && is_packed4(tx) && is_packed4(tdt) && is_packed4(ta) && is_packed4(d), "s, x, dt, A and dst must be contiguous");
    B200_REQUIRE(tb.nb[0] == 4 && tc.nb[0] == 4, "B and C must be contiguous along dim 0");
    const int64_t d_state = ts.ne[0], d_inner = ts.ne[1], n_t = tx.ne[1], n_s = ts.ne[2];
    B200_REQUIRE(ts.ne[3] == 1 && tx.ne[3] == 1 && tb.ne[3] == 1 && ta.ne[2] == 1 && ta.ne[3] == 1, "s, x and B must be 3-D, A a matrix");
    // what the CPU backend asserts beyond contiguity (it also holds where a dimension is 1): the strides dst's layout is built from
    B200_REQUIRE(ts.nb[0] == 4 && tx.nb[0] == 4 && tdt.nb[0] == 4 && ta.nb[0] == 4 && ts.nb[1] == (size_t)d_state * 4 &&
                 ts.nb[2] == (size_t)(d_state * d_inner) * 4 && tx.nb[3] == (size_t)nelem(tx) * 4, "s and x must have packed strides");
    B200_REQUIRE(tx.ne[0] == d_inner && tx.ne[2] == n_s, "x must be [d_inner, n_t, n_s]");
    B200_REQUIRE(same_shape(tdt, tx) && same_shape(tc, tb), "dt must have x's shape and C B's");
    B200_REQUIRE(ta.ne[0] == d_state && ta.ne[1] == d_inner, "A must be [d_state, d_inner]");
    B200_REQUIRE(tb.ne[0] == d_state && tb.ne[1] == n_t && tb.ne[2] == n_s, "B and C must be [d_state, n_t, n_s]");
    B200_REQUIRE(nelem(d) == nelem(tx) + nelem(ts), "dst must hold y and the final states");
    if (d_inner == 0 || n_s == 0) return accepted;
    B200_REQUIRE(n_s <= 65535 && (d_inner + 127) / 128 <= 0x7fffffff, "too many rows / sequences for one grid");
    return accepted;
}

// what RWKV_WKV6 and GATED_LINEAR_ATTN share: k, v, a (r or q) and b (td or g) f32 [S, H, T], the state s f32 with S S H n_seqs elements
// (n_seqs = its ne1, as ggml reads it) and dst f32 [S H, T + S n_seqs].  ggml-cpu indexes every one of them flat, whatever its strides,
// so all must be packed.
inline op_check check_wkv_common(const ggml_b200_tensor * k, const ggml_b200_tensor * v, const ggml_b200_tensor * a, const ggml_b200_tensor * b,
                                 const ggml_b200_tensor * s, const ggml_b200_tensor * dst) {
    B200_REQUIRE(k && v && a && b && s && dst, "all sources and dst are required");
    B200_REQUIRE(k->type == F32 && v->type == F32 && a->type == F32 && b->type == F32 && s->type == F32 && dst->type == F32, "all tensors must be f32");
    B200_REQUIRE(is_packed4(*k) && is_packed4(*v) && is_packed4(*a) && is_packed4(*b) && is_packed4(*s) && is_packed4(*dst), "all tensors must be contiguous");
    const int64_t S = k->ne[0], H = k->ne[1], T = k->ne[2], n_seqs = s->ne[1];
    B200_REQUIRE(k->ne[3] == 1 && H >= 1, "k must be [S, H, T] with at least one head");
    B200_REQUIRE(same_shape(*v, *k) && same_shape(*a, *k) && same_shape(*b, *k), "v and r / q and td / g must have k's shape");
    B200_REQUIRE(nelem(*s) == S * S * H * n_seqs, "the state must hold S * S * H * n_seqs values (n_seqs = its ne1)");
    B200_REQUIRE(dst->ne[0] == S * H && dst->ne[1] == T + S * n_seqs && dst->ne[2] == 1 && dst->ne[3] == 1, "dst must be [S * H, T + S * n_seqs]");
    B200_REQUIRE(S <= WKV_MAX_HEAD, "head size above 256");
    if (T == 0) return accepted;                           // ggml-cpu writes nothing
    // ggml-cpu gives each sequence T / n_seqs tokens and divides by that count
    B200_VALID(n_seqs >= 1 && T % n_seqs == 0, "the tokens must split evenly over the sequences (T % n_seqs == 0)");
    if (S == 0) return accepted;
    B200_REQUIRE(H <= 65535 && n_seqs <= 65535, "too many heads / sequences for one grid");
    return accepted;
}

inline op_check check_rwkv_wkv6(const ggml_b200_tensor * k, const ggml_b200_tensor * v, const ggml_b200_tensor * r, const ggml_b200_tensor * tf,
                                const ggml_b200_tensor * td, const ggml_b200_tensor * s, const ggml_b200_tensor * dst) {
    B200_REQUIRE(tf, "tf is required");
    B200_REQUIRE(tf->type == F32 && is_packed4(*tf), "tf must be f32 and contiguous");
    if (k) B200_REQUIRE(nelem(*tf) == k->ne[0] * k->ne[1], "tf must hold S * H values");
    return check_wkv_common(k, v, r, td, s, dst);
}

inline op_check check_gated_linear_attn(const ggml_b200_tensor * k, const ggml_b200_tensor * v, const ggml_b200_tensor * q, const ggml_b200_tensor * g,
                                        const ggml_b200_tensor * s, const ggml_b200_tensor * dst) {
    return check_wkv_common(k, v, q, g, s, dst);
}

// IM2COL: src0 the conv kernel (its extents), src1 the f32 input, dst [IC KH KW, OW, OH, N] (1-D: [IC KW, OW, N, 1]), f32 or f16
inline op_check check_im2col(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, const ggml_b200_im2col_params * params) {
    B200_REQUIRE(src0 && src1 && dst && params, "src0, src1, dst and params are required");
    const ggml_b200_tensor & k = *src0, & x = *src1, & d = *dst;
    const ggml_b200_im2col_params & c = *params;
    B200_VALID(c.is_2D == 0 || c.is_2D == 1, "is_2D must be 0 or 1");
    B200_VALID(c.s0 >= 1 && c.d0 >= 1 && (!c.is_2D || (c.s1 >= 1 && c.d1 >= 1)), "strides and dilations must be >= 1");
    B200_REQUIRE(x.type == F32 && x.nb[0] == 4, "src1 must be f32, contiguous along dim 0");
    // ggml-cpu writes dst as if it were packed, whatever its strides
    B200_REQUIRE(is_float(d.type) && is_packed(d, d.type == F32 ? 4 : 2), "dst must be f32 or f16 and packed");
    B200_REQUIRE(d.type == F32 || (k.type == F16 && k.nb[0] == 2), "an f16 dst needs an f16 src0");
    B200_REQUIRE(c.is_2D || x.ne[3] == 1, "the 1-D input must be 3-D");
    const bool two = c.is_2D == 1;
    const int64_t KW = k.ne[0], KH = two ? k.ne[1] : 1, IC = two ? x.ne[2] : x.ne[1], N = two ? x.ne[3] : x.ne[2];
    const int64_t OW = conv_out_size(x.ne[0], KW, c.s0, c.p0, c.d0), OH = two ? conv_out_size(x.ne[1], KH, c.s1, c.p1, c.d1) : 1;
    B200_REQUIRE(d.ne[0] == IC * KH * KW && d.ne[1] == OW && d.ne[2] == (two ? OH : N) && d.ne[3] == (two ? N : 1),
                 "dst must be [IC KH KW, OW, OH, N] (1-D: [IC KW, OW, N, 1]) of the input and params");
    // ggml-cpu keeps the image and channel offsets of src1 in an int: beyond INT32_MAX the two backends would read different data
    B200_REQUIRE((two ? x.nb[3] : x.nb[2]) <= 0x7fffffff && (two ? x.nb[2] : x.nb[1]) <= 0x7fffffff, "src1 image / channel strides above INT32_MAX bytes");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE((nelem(d) + 255) / 256 <= 0x7fffffff, "too many elements for one grid");
    return accepted;
}

// POOL_2D: src f32 [IW, IH, C, N] (elements packed along dim 0), dst f32 [OW, OH, C, N] packed; OW / OH are dst's (ggml_pool_2d derives them
// from float paddings), so only C and N are compared with src
inline op_check check_pool_2d(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, const ggml_b200_pool_params * params) {
    B200_REQUIRE(src && dst && params, "src, dst and params are required");
    const ggml_b200_tensor & s = *src, & d = *dst;
    const ggml_b200_pool_params & p = *params;
    B200_VALID(p.op == 0 || p.op == 1, "op must be 0 (MAX) or 1 (AVG): ggml-cpu aborts on POOL_COUNT");
    B200_VALID(p.k0 >= 1 && p.k1 >= 1 && p.s0 >= 1 && p.s1 >= 1, "window and stride must be >= 1");
    B200_REQUIRE(s.type == F32 && d.type == F32, "src and dst must be f32");
    B200_REQUIRE(s.nb[0] == 4, "src must be contiguous along dim 0");
    // ggml-cpu writes dst as if it were packed, whatever its strides
    B200_REQUIRE(is_packed4(d), "dst must be packed");
    B200_VALID(d.ne[2] == s.ne[2] && d.ne[3] == s.ne[3] && d.ne[0] >= 0 && d.ne[1] >= 0, "dst must be [OW, OH, C, N] of src's C and N");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE((nelem(d) + 255) / 256 <= 0x7fffffff, "too many elements for one grid");
    return accepted;
}

// UPSCALE (nearest): src and dst f32, any strides; ggml_upscale_ext asserts dst extents >= src's
inline op_check check_upscale(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src && dst, "src and dst are required");
    const ggml_b200_tensor & s = *src, & d = *dst;
    B200_REQUIRE(s.type == F32 && d.type == F32, "src and dst must be f32");
    if (nelem(d) == 0) return accepted;
    B200_VALID(s.ne[0] >= 1 && s.ne[1] >= 1 && s.ne[2] >= 1 && s.ne[3] >= 1, "src must not be empty");
    B200_VALID(d.ne[0] >= s.ne[0] && d.ne[1] >= s.ne[1] && d.ne[2] >= s.ne[2] && d.ne[3] >= s.ne[3], "dst extents must be >= src's");
    B200_REQUIRE((nelem(d) + 255) / 256 <= 0x7fffffff, "too many elements for one grid");
    return accepted;
}

// LEAKY_RELU: src and dst f32 of one shape, elements packed along dim 0 (dst may be src: in place)
inline op_check check_leaky_relu(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src && dst, "src and dst are required");
    const ggml_b200_tensor & s = *src, & d = *dst;
    B200_REQUIRE(s.type == F32 && d.type == F32, "src and dst must be f32");
    B200_REQUIRE(s.nb[0] == 4 && d.nb[0] == 4, "src and dst must be contiguous along dim 0");
    B200_VALID(same_shape(s, d), "src and dst shapes differ");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE((nelem(d) + 255) / 256 <= 0x7fffffff, "too many elements for one grid");
    return accepted;
}

// the element size of a type REPEAT moves as raw words, 0 for any other: the types ggml-cpu repeats
inline size_t repeat_elem_size(int32_t t) {
    switch (t) {
        case GGML_B200_TYPE_F32: case GGML_B200_TYPE_I32: return 4;
        case GGML_B200_TYPE_F16: case GGML_B200_TYPE_BF16: case GGML_B200_TYPE_I16: return 2;
        default: return 0;
    }
}

// REPEAT: src and dst of one 4- or 2-byte type, both contiguous along dim 0 (ggml-cpu asserts so), dst a whole repeat of src
inline op_check check_repeat(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src && dst, "src and dst are required");
    const ggml_b200_tensor & s = *src, & d = *dst;
    const size_t es = repeat_elem_size(s.type);
    B200_REQUIRE(es && d.type == s.type, "src and dst must be one type of f32, i32, f16, bf16 or i16");
    B200_REQUIRE(s.nb[0] == es && d.nb[0] == es, "src and dst must be contiguous along dim 0");
    // ggml_can_repeat: an empty src repeats only into an empty dst
    if (nelem(s) == 0) { B200_VALID(nelem(d) == 0, "an empty src repeats only into an empty dst"); return accepted; }
    B200_VALID(d.ne[0] % s.ne[0] == 0 && d.ne[1] % s.ne[1] == 0 && d.ne[2] % s.ne[2] == 0 && d.ne[3] % s.ne[3] == 0,
               "dst extents must be whole multiples of src's");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE((nelem(d) + 255) / 256 <= 0x7fffffff, "too many elements for one grid");
    return accepted;
}

// WIN_PART / WIN_UNPART / GET_REL_POS / ADD_REL_POS (b200_sam.cuh): one CTA row of threads per row of ne0 elements, rows on grid x (32-bit
// row indices), blocks of a row on grid y
inline bool rows_fit_grid(int64_t rows, int64_t row_len) { return rows <= 0x7fffffff && (row_len + 255) / 256 <= 65535; }
inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// WIN_PART: src f32 [C, W0, H0, 1] -> dst f32 [C, w, w, npx npy], both packed (ggml-cpu indexes them as packed); op_params npx, npy, w as
// ggml_win_part derives them
inline op_check check_win_part(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t npx, int32_t npy, int32_t w) {
    B200_REQUIRE(src && dst, "src and dst are required");
    const ggml_b200_tensor & s = *src, & d = *dst;
    B200_REQUIRE(s.type == GGML_B200_TYPE_F32 && d.type == GGML_B200_TYPE_F32, "src and dst must be f32");
    B200_REQUIRE(is_packed4(s) && is_packed4(d), "src and dst must be packed");
    B200_VALID(w >= 1, "the window must be >= 1");
    B200_VALID(s.ne[3] == 1, "src must be one image [C, W0, H0, 1]");
    B200_VALID(npx == ceil_div(s.ne[1], w) && npy == ceil_div(s.ne[2], w), "npx / npy must be ceil(W0 / w) / ceil(H0 / w)");
    B200_VALID(d.ne[0] == s.ne[0] && d.ne[1] == w && d.ne[2] == w && d.ne[3] == (int64_t)npx * npy, "dst must be [C, w, w, npx npy]");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE(rows_fit_grid(nrows(d), d.ne[0]) && s.ne[1] * s.ne[2] <= 0x7fffffff, "too many rows for one grid");
    return accepted;
}

// WIN_UNPART: src f32 [C, w, w, np] -> dst f32 [C, W0, H0, 1], both packed; np must hold every window of the image, or the reads leave src
inline op_check check_win_unpart(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t w) {
    B200_REQUIRE(src && dst, "src and dst are required");
    const ggml_b200_tensor & s = *src, & d = *dst;
    B200_REQUIRE(s.type == GGML_B200_TYPE_F32 && d.type == GGML_B200_TYPE_F32, "src and dst must be f32");
    B200_REQUIRE(is_packed4(s) && is_packed4(d), "src and dst must be packed");
    B200_VALID(w >= 1, "the window must be >= 1");
    B200_VALID(d.ne[0] == s.ne[0] && d.ne[3] == 1 && s.ne[1] == w && s.ne[2] == w, "src must be [C, w, w, np] and dst [C, W0, H0, 1]");
    B200_VALID(s.ne[3] >= ceil_div(d.ne[1], w) * ceil_div(d.ne[2], w), "src must hold ceil(W0 / w) ceil(H0 / w) windows");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE(rows_fit_grid(nrows(d), d.ne[0]) && nrows(s) <= 0x7fffffff, "too many rows for one grid");
    return accepted;
}

// GET_REL_POS: src f16 [C, 2w - 1] -> dst f16 [C, w, w], both packed (ggml-cpu reads src row p at p ne0).  ggml-cpu also runs a BF16 src
// into its F16 dst as raw bits; nothing builds that, and it is declined.
inline op_check check_get_rel_pos(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src && dst, "src and dst are required");
    const ggml_b200_tensor & s = *src, & d = *dst;
    B200_REQUIRE(s.type == GGML_B200_TYPE_F16 && d.type == GGML_B200_TYPE_F16, "src and dst must be f16");
    B200_REQUIRE(is_packed(s, 2) && is_packed(d, 2), "src and dst must be packed");
    const int64_t w = d.ne[1];
    B200_VALID(w >= 1 && d.ne[2] == w && d.ne[3] == 1 && d.ne[0] == s.ne[0] && s.ne[1] == 2 * w - 1 && s.ne[2] == 1 && s.ne[3] == 1,
               "src must be [C, 2w - 1] and dst [C, w, w]");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE(rows_fit_grid(nrows(d), d.ne[0]), "too many rows for one grid");
    return accepted;
}

// ADD_REL_POS: src0 and dst f32 [L L, A B, P, 1], pw = src1 and ph = src2 f32 [L, A, B, P], all packed (ggml_add_rel_pos asserts it, and
// ggml-cpu indexes them so); dst may be src0 (in place).  ggml-cpu touches only the first slice of a src0 with ne3 > 1: declined.
inline op_check check_add_rel_pos(const ggml_b200_tensor * src0, const ggml_b200_tensor * pw, const ggml_b200_tensor * ph, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src0 && pw && ph && dst, "src0, pw, ph and dst are required");
    const ggml_b200_tensor & a = *src0, & w = *pw, & h = *ph, & d = *dst;
    B200_REQUIRE(a.type == GGML_B200_TYPE_F32 && w.type == GGML_B200_TYPE_F32 && h.type == GGML_B200_TYPE_F32 && d.type == GGML_B200_TYPE_F32,
                 "src0, pw, ph and dst must be f32");
    B200_REQUIRE(is_packed4(a) && is_packed4(w) && is_packed4(h) && is_packed4(d), "src0, pw, ph and dst must be packed");
    B200_REQUIRE(a.ne[3] == 1, "src0 must have ne3 == 1 (ggml-cpu adds to its first slice only)");
    B200_VALID(same_shape(w, h) && same_shape(a, d), "pw and ph, src0 and dst must have one shape each");
    const int64_t L = w.ne[0];
    B200_VALID(a.ne[0] == L * L && a.ne[1] == w.ne[1] * w.ne[2] && a.ne[2] == w.ne[3], "src0 must be [L L, A B, P] of pw's [L, A, B, P]");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE(rows_fit_grid(nrows(d), d.ne[0]), "too many rows for one grid");
    return accepted;
}

// CONV_TRANSPOSE_2D (ggml_conv_transpose_2d_p0): kernel f16 [Kw, Kh, Cout, Cin] with packed Kw x Kh planes, input f32 [W, H, Cin, 1]
// contiguous along dim 0, dst f32 [(W-1) s + Kw, (H-1) s + Kh, Cout, 1] packed: the layouts ggml-cpu reads.  ggml-cpu computes only the
// first image of a batch (and leaves the rest zero): ne3 > 1 is declined.
inline op_check check_conv_transpose_2d(const ggml_b200_tensor * kernel, const ggml_b200_tensor * input, const ggml_b200_tensor * dst, int32_t stride) {
    B200_REQUIRE(kernel && input && dst, "kernel, input and dst are required");
    const ggml_b200_tensor & k = *kernel, & x = *input, & d = *dst;
    B200_REQUIRE(k.type == GGML_B200_TYPE_F16 && x.type == GGML_B200_TYPE_F32 && d.type == GGML_B200_TYPE_F32, "kernel f16, input and dst f32");
    B200_REQUIRE(k.nb[0] == 2 && k.nb[1] == (size_t)(2 * k.ne[0]), "the kernel's Kw x Kh planes must be packed");
    B200_REQUIRE(x.nb[0] == 4, "input must be contiguous along dim 0");
    B200_REQUIRE(is_packed4(d), "dst must be packed");
    B200_REQUIRE(x.ne[3] == 1 && d.ne[3] == 1, "one image only (ggml-cpu computes the first image of a batch)");
    B200_VALID(stride >= 1, "stride must be >= 1");
    B200_VALID(k.ne[3] == x.ne[2] && d.ne[2] == k.ne[2], "kernel must be [Kw, Kh, Cout, Cin] of input's Cin and dst's Cout");
    B200_VALID(d.ne[0] == (x.ne[0] - 1) * stride + k.ne[0] && d.ne[1] == (x.ne[1] - 1) * stride + k.ne[1],
               "dst must be [(W-1) s + Kw, (H-1) s + Kh, Cout]");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE(stride <= 255, "stride must be <= 255 (one grid z per stride phase)");
    B200_REQUIRE(d.ne[0] <= 0x7fffffff && d.ne[1] <= 0x7fffffff && k.ne[2] <= 0x7fffffff && k.ne[3] <= 0x7fffffff, "extents must fit 32 bits");
    B200_REQUIRE(ceil_div(ceil_div(d.ne[0], stride), 32) * ceil_div(ceil_div(d.ne[1], stride), 2) <= 0x7fffffff && ceil_div(k.ne[2], 32) <= 65535,
                 "too many tiles for one grid");
    return accepted;
}

// ------------------------------------------------------------------ the ops of ggml_opt's backward and optimizer graphs (b200_train.cuh)

// OUT_PROD: src0 f32 [ne0, K, ne02, ne03] contiguous along dim 0, src1 f32 [ne1, K, ne2, ne3] any strides, dst f32 packed (ggml-cpu zeroes it
// as packed); ne2 % ne02 == 0, ne3 % ne03 == 0.  ggml-cpu's f16 and quantized src0 forms are declined.
inline op_check check_out_prod(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src0 && src1 && dst, "src0, src1 and dst are required");
    const ggml_b200_tensor & a = *src0, & b = *src1, & d = *dst;
    B200_REQUIRE(a.type == F32 && b.type == F32 && d.type == F32, "src0, src1 and dst must be f32");
    B200_REQUIRE(a.nb[0] == 4, "src0 must be contiguous along dim 0");
    B200_REQUIRE(is_packed4(d), "dst must be packed");
    B200_VALID(d.ne[0] == a.ne[0] && d.ne[1] == b.ne[0] && a.ne[1] == b.ne[1] && d.ne[2] == b.ne[2] && d.ne[3] == b.ne[3],
               "dst must be [src0 ne0, src1 ne0, src1 ne2, src1 ne3] and src0, src1 share K");
    B200_VALID(a.ne[2] >= 1 && a.ne[3] >= 1 && d.ne[2] % a.ne[2] == 0 && d.ne[3] % a.ne[3] == 0, "src0's batch dims must divide dst's");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE((d.ne[1] + 127) / 128 <= 65535 && d.ne[2] * d.ne[3] <= 65535 && (d.ne[0] + 127) / 128 <= 0x7fffffff, "too many tiles for one grid");
    return accepted;
}

// CROSS_ENTROPY_LOSS: logits and labels f32 of one shape, rows contiguous along dim 0 (ggml-cpu reads row i1 at i1 nb1: evenly spaced rows
// are the caller's condition), dst an f32 scalar
inline op_check check_cross_entropy_loss(const ggml_b200_tensor * logits, const ggml_b200_tensor * labels, const ggml_b200_tensor * dst) {
    B200_REQUIRE(logits && labels && dst, "logits, labels and dst are required");
    const ggml_b200_tensor & x = *logits, & l = *labels, & d = *dst;
    B200_REQUIRE(x.type == F32 && l.type == F32 && d.type == F32, "logits, labels and dst must be f32");
    B200_REQUIRE(x.nb[0] == 4 && l.nb[0] == 4, "rows must be contiguous along dim 0");
    B200_VALID(same_shape(x, l), "logits and labels must have one shape");
    B200_VALID(nelem(d) == 1, "dst must be a scalar");
    return accepted;
}

// CROSS_ENTROPY_LOSS_BACK: grad an f32 scalar, logits, labels and dst f32 of one shape, all packed (ggml-cpu asserts it)
inline op_check check_cross_entropy_loss_back(const ggml_b200_tensor * grad, const ggml_b200_tensor * logits, const ggml_b200_tensor * labels,
                                              const ggml_b200_tensor * dst) {
    B200_REQUIRE(grad && logits && labels && dst, "grad, logits, labels and dst are required");
    const ggml_b200_tensor & g = *grad, & x = *logits, & l = *labels, & d = *dst;
    B200_REQUIRE(g.type == F32 && x.type == F32 && l.type == F32 && d.type == F32, "grad, logits, labels and dst must be f32");
    B200_REQUIRE(is_packed4(x) && is_packed4(l) && is_packed4(d), "logits, labels and dst must be packed");
    B200_VALID(nelem(g) == 1, "grad must be a scalar");
    B200_VALID(same_shape(x, l) && same_shape(x, d), "logits, labels and dst must have one shape");
    if (nelem(d) == 0) return accepted;
    B200_REQUIRE(nrows(d) <= 0x7fffffff, "too many rows for one grid");
    return accepted;
}

// OPT_STEP_ADAMW: w, g, m, v f32 of one shape, all packed (ggml-cpu addresses g, m and v with w's offsets), params f32 with 7 elements
inline op_check check_opt_step_adamw(const ggml_b200_tensor * w, const ggml_b200_tensor * g, const ggml_b200_tensor * m, const ggml_b200_tensor * v,
                                     const ggml_b200_tensor * params) {
    B200_REQUIRE(w && g && m && v && params, "w, g, m, v and params are required");
    B200_REQUIRE(w->type == F32 && g->type == F32 && m->type == F32 && v->type == F32 && params->type == F32, "w, g, m, v and params must be f32");
    B200_REQUIRE(is_packed4(*w) && is_packed4(*g) && is_packed4(*m) && is_packed4(*v) && is_packed4(*params), "w, g, m, v and params must be packed");
    B200_VALID(same_shape(*w, *g) && same_shape(*w, *m) && same_shape(*w, *v), "w, g, m and v must have one shape");
    B200_VALID(nelem(*params) == 7, "params must hold 7 values");
    return accepted;
}

// ARGMAX: src f32 [ne0, ne1] rows contiguous along dim 0, dst i32 [ne1] contiguous along dim 0
inline op_check check_argmax(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src && dst, "src and dst are required");
    const ggml_b200_tensor & s = *src, & d = *dst;
    B200_REQUIRE(s.type == F32 && d.type == I32, "src must be f32, dst i32");
    B200_REQUIRE(s.nb[0] == 4 && d.nb[0] == 4, "src rows and dst must be contiguous along dim 0");
    B200_VALID(s.ne[2] == 1 && s.ne[3] == 1 && d.ne[0] == s.ne[1] && d.ne[1] == 1 && d.ne[2] == 1 && d.ne[3] == 1, "src must be a matrix, dst [ne1]");
    if (s.ne[1] == 0) return accepted;
    B200_VALID(s.ne[0] >= 1, "rows must not be empty");
    B200_REQUIRE(s.ne[0] <= 0x7fffffff && s.ne[1] <= 0x7fffffff, "extents must fit 32 bits");
    return accepted;
}

// COUNT_EQUAL: src0 and src1 i32 of one shape, any strides, dst an i64 scalar.  ggml-cpu's row walk (ggml-cpu.c:5850-5853) names the right
// row only when ne2 == ne3 == 1: others are declined.
inline op_check check_count_equal(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src0 && src1 && dst, "src0, src1 and dst are required");
    const ggml_b200_tensor & a = *src0, & b = *src1, & d = *dst;
    B200_REQUIRE(a.type == I32 && b.type == I32 && d.type == GGML_B200_TYPE_I64, "src0 and src1 must be i32, dst i64");
    B200_VALID(same_shape(a, b), "src0 and src1 must have one shape");
    B200_VALID(nelem(d) == 1, "dst must be a scalar");
    B200_REQUIRE(a.ne[2] == 1 && a.ne[3] == 1, "ne2 and ne3 must be 1 (the CPU backend's row walk)");
    return accepted;
}

// SUM: src f32 contiguous along dim 0 (ggml-cpu asserts it), any other strides, dst an f32 scalar
inline op_check check_sum(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src && dst, "src and dst are required");
    B200_REQUIRE(src->type == F32 && dst->type == F32, "src and dst must be f32");
    B200_REQUIRE(src->nb[0] == 4, "src must be contiguous along dim 0");
    B200_VALID(nelem(*dst) == 1, "dst must be a scalar");
    return accepted;
}

// REPEAT_BACK: src and dst f32, both contiguous along dim 0 (ggml-cpu asserts nb0 == nb00 == 4 and honours every other stride), every src
// extent a whole multiple of dst's.  ggml-cpu has no other type (it aborts on I32 / I16): declined.
inline op_check check_repeat_back(const ggml_b200_tensor * src, const ggml_b200_tensor * dst) {
    B200_REQUIRE(src && dst, "src and dst are required");
    const ggml_b200_tensor & s = *src, & d = *dst;
    B200_REQUIRE(s.type == F32 && d.type == F32, "src and dst must be f32");
    B200_REQUIRE(s.nb[0] == 4 && d.nb[0] == 4, "src and dst must be contiguous along dim 0");
    if (nelem(d) == 0) return accepted;
    for (int i = 0; i < 4; ++i) B200_VALID(s.ne[i] % d.ne[i] == 0, "every src extent must be a whole multiple of dst's");
    return accepted;
}

#undef B200_REQUIRE
#undef B200_VALID

} // namespace b200
