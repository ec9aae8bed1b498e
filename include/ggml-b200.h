/* ggml-b200.h — the C ABI of the B200-native ggml backend.
 *
 * Two layers, both plain C (pointers, sizes, an opaque stream handle; no torch / ggml C++ types):
 *
 *  (1) KERNEL-LAUNCH SHIM  — libggml-b200-kernels.so.  Hand-written sm_90a kernels for the hot path
 *      GGML_OP_MUL_MAT / GGML_OP_MUL_MAT_ID over block-quantized weights + their dequantize family.
 *      Replaces, in the reference (paths relative to the ggml tree @ 9a4acb37):
 *        ggml_cuda_op_mul_mat_vec_q   src/ggml-cuda/mmvq.cu:338      (quantized GEMV, n <= 8)
 *        ggml_cuda_op_mul_mat_q       src/ggml-cuda/mmq.cu:3         (quantized GEMM)
 *        quantize_row_q8_1_cuda       src/ggml-cuda/quantize.cu:129  (activation quantizer)
 *        ggml_cuda_mul_mat_id         src/ggml-cuda/ggml-cuda.cu:1955
 *        dequantize_row_*_cuda        src/ggml-cuda/convert.cu:500-640
 *      and computes what the CPU backend's ggml_compute_forward_mul_mat (src/ggml-cpu/ggml-cpu.c:7428)
 *      and ggml_compute_forward_mul_mat_id (:7609) compute.
 *
 *  (2) BACKEND PLUG-IN     — libggml-b200.so.  The reference's own backend SPI
 *      (src/ggml-backend-impl.h: ggml_backend_reg_i / _device_i / _buffer_type_i / _buffer_i / ggml_backend_i)
 *      implemented on top of (1), so ggml_backend_sched, tests/test-backend-ops and examples/gpt-2 run
 *      unmodified.  Entry points: ggml_backend_init / ggml_backend_score (dynamic loading,
 *      src/ggml-backend-reg.cpp:220-263), ggml_backend_b200_reg / ggml_backend_b200_init, and the
 *      include/ggml-cuda.h:23-45 facade (ggml_backend_cuda_init …) for programs compiled with -DGGML_USE_CUDA.
 *
 * All device pointers are CUDA device pointers on the current device; `stream` is a cudaStream_t
 * (CUstream) cast to void*; functions are asynchronous on that stream unless stated otherwise.
 * Return value: 0 on success, a negative GGML_B200_E* code otherwise (never a silent CPU fallback).
 */
#ifndef GGML_B200_H
#define GGML_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#  define GGML_B200_API __declspec(dllexport)
#else
#  define GGML_B200_API __attribute__((visibility("default")))
#endif

enum ggml_b200_status {
    GGML_B200_OK            =  0,
    GGML_B200_EUNSUPPORTED  = -1,  /* type / shape combination not implemented */
    GGML_B200_EINVAL        = -2,  /* malformed arguments (K not a multiple of the block size, NULL pointers, …) */
    GGML_B200_EWORKSPACE    = -3,  /* workspace too small: call ggml_b200_mul_mat_workspace_size */
    GGML_B200_ECUDA         = -4,  /* CUDA runtime error, see ggml_b200_last_error */
};

/* numeric ids are the reference's enum ggml_type (include/ggml.h:351-390) */
enum ggml_b200_type {
    GGML_B200_TYPE_F32  = 0,  GGML_B200_TYPE_F16  = 1,
    GGML_B200_TYPE_Q4_0 = 2,  GGML_B200_TYPE_Q8_0 = 8,
    GGML_B200_TYPE_Q4_K = 12, GGML_B200_TYPE_Q5_K = 13, GGML_B200_TYPE_Q6_K = 14,
    /* next formats (SURVEY 8f-2): generic mat-vec, MUL_MAT_ID and dequantize kernels only; block layouts src/ggml-common.h:168-203, 247-276 */
    GGML_B200_TYPE_Q4_1 = 3,  GGML_B200_TYPE_Q5_0 = 6,  GGML_B200_TYPE_Q5_1 = 7, GGML_B200_TYPE_Q2_K = 10, GGML_B200_TYPE_Q3_K = 11, GGML_B200_TYPE_IQ4_NL = 20, GGML_B200_TYPE_IQ4_XS = 23,
    /* grid-codebook i-quants (src/ggml-common.h:330-396; codebooks extracted from it at build time): generic mat-vec, MUL_MAT_ID, dequantize */
    GGML_B200_TYPE_IQ2_XXS = 16, GGML_B200_TYPE_IQ3_XXS = 18, GGML_B200_TYPE_IQ1_S = 19,
    GGML_B200_TYPE_IQ2_XS = 17, GGML_B200_TYPE_IQ3_S = 21, GGML_B200_TYPE_IQ2_S = 22, GGML_B200_TYPE_IQ1_M = 29, GGML_B200_TYPE_TQ1_0 = 34, GGML_B200_TYPE_TQ2_0 = 35,
};

/* ---------------------------------------------------------------------------------------------
 * MUL_MAT:  dst[i3][i2][n][m] = sum_k src0[i3/r3][i2/r2][m][k] * src1[i3][i2][n][k]
 * with ggml's shapes/strides (src/ggml.c:2686-2709): src0 = W[ne00=K, ne01=M, ne02, ne03] in a
 * block-quantized type (rows contiguous along K, strides nb01/nb02/nb03 in BYTES), src1 = X[K, N, ne12, ne13]
 * f32 (element stride 4 B along K, nb11/nb12/nb13 in bytes), dst = Y[M, N, ne12, ne13] f32 contiguous.
 * Broadcast: ne12 % ne02 == 0, ne13 % ne03 == 0.
 * ------------------------------------------------------------------------------------------- */
typedef struct ggml_b200_mul_mat_args {
    int32_t      type;                    /* enum ggml_b200_type of src0 */
    int32_t      flags;                   /* GGML_B200_MM_* */
    int64_t      K, M, N;                 /* ne00, ne01, ne11 */
    int64_t      ne02, ne03, ne12, ne13;  /* batch dims (>= 1) */
    size_t       nb01, nb02, nb03;        /* src0 strides, bytes */
    size_t       nb11, nb12, nb13;        /* src1 strides, bytes */
    const void * src0;                    /* device, packed blocks */
    const float* src1;                    /* device */
    float *      dst;                     /* device, contiguous [ne13][ne12][N][M] */
    void *       workspace;               /* device scratch, >= ggml_b200_mul_mat_workspace_size() */
    size_t       workspace_size;
} ggml_b200_mul_mat_args;

enum {
    GGML_B200_MM_AUTO        = 0,
    GGML_B200_MM_FORCE_GENERIC = 1,   /* strided one-warp-per-output kernel (any shape) */
    GGML_B200_MM_FORCE_GEMV  = 2,     /* TMA-staged bandwidth kernel (N <= 8) */
    GGML_B200_MM_FORCE_GEMM  = 4,     /* tensor-core (wgmma) kernel */
    GGML_B200_MM_SRC0_STATIC = 16,    /* src0 is not written by the preceding kernel on this stream (model weights): the mat-vec may
                                         prefetch it before waiting for that kernel (programmatic dependent launch) */
    GGML_B200_MM_SRC1_STATIC = 32,    /* src1 is not written by ANY kernel still in flight on this stream (inputs that were final before the
                                         sequence of launches began, e.g. a perf harness repeating an op on fixed inputs), and dst is not
                                         read or written by any of them: the launch never waits for its predecessors before computing, so
                                         independent mat-vecs overlap.  It still waits for them before it retires, so completion stays
                                         ordered along the stream.  NOT valid for "the kernel before the previous one produced src1". */
    GGML_B200_MM_GEMV_V1     = 8,     /* with FORCE_GEMV: the first-generation 64-weight-unit kernel (mmvq.cu) even for n = 1 */
    GGML_B200_MM_GEMV_MMA    = 64,    /* bandwidth path: the int8 mma.sync consume kernel (mmvq_mma.cu; default for 2 <= n <= 8) also for n = 1 */
    GGML_B200_MM_GEMV_DP4A   = 128,   /* bandwidth path: the dp4a task-dot kernel (mmvq_sb.cu; default for n = 1) also for 2 <= n <= 8 */
};

GGML_B200_API size_t ggml_b200_mul_mat_workspace_size(const ggml_b200_mul_mat_args * args);
GGML_B200_API int    ggml_b200_mul_mat(const ggml_b200_mul_mat_args * args, void * stream);
/* which kernel family AUTO would pick: 1 generic, 2 gemv, 4 gemm, <0 error */
GGML_B200_API int    ggml_b200_mul_mat_plan(const ggml_b200_mul_mat_args * args);

/* MUL_MAT whose two following ggml nodes are folded into the kernel's epilogue: dst_bias = dst + bias (GGML_OP_ADD with a [M] f32
 * bias) and, if unary == 1, dst_unary = GELU(dst_bias) (GGML_UNARY_OP_GELU); all three tensors are written, so the graph's other
 * readers still see them.  Returns GGML_B200_EUNSUPPORTED when the shape does not run on the n = 1 mat-vec kernel (caller falls back
 * to separate ops). */
typedef struct ggml_b200_epilogue {
    const float * bias;       /* [M] */
    float *       dst_bias;   /* [M] */
    int32_t       unary;      /* 0 none, 1 GELU, 2 residual add: dst_unary = dst_bias + residual (a second GGML_OP_ADD, e.g. the skip connection) */
    float *       dst_unary;  /* [M] or NULL */
    const float * residual;   /* [M], unary == 2 only; may alias dst_unary */
} ggml_b200_epilogue;
/* dense fp16 weights [M][K] (row stride nb01 bytes, a multiple of 16) x f32 activations [N][K] -> f32 [N][M] on the tensor cores, n >= 9, K % 256 == 0
   (the reference: cuBLAS GEMM, src/ggml-cuda/ggml-cuda.cu:1158-1300).  workspace_size = 0 from the size function: shape not eligible. */
GGML_B200_API size_t ggml_b200_mul_mat_f16_workspace_size(int64_t M, int64_t N, int64_t K);
GGML_B200_API int    ggml_b200_mul_mat_f16(const void * w, size_t nb01, const float * x, size_t nb11, float * y, int64_t M, int64_t N, int64_t K,
                                           void * workspace, size_t workspace_size, uint32_t flags, void * stream);
GGML_B200_API int    ggml_b200_mul_mat_fused(const ggml_b200_mul_mat_args * args, const ggml_b200_epilogue * epilogue, void * stream);

/* MUL_MAT with HOST activations / results: copies src1 (host, contiguous [N][K]) to the device, runs
 * ggml_b200_mul_mat and copies dst back, all on `stream`, then synchronizes it.  src0 stays device-resident
 * (weights are uploaded once at model load, like the reference's buffer.set_tensor).  Used for the
 * end-to-end measurement; `args->src1` / `args->dst` must point at device staging buffers. */
GGML_B200_API int    ggml_b200_mul_mat_host(const ggml_b200_mul_mat_args * args, const float * host_src1, float * host_dst, void * stream);
/* n MUL_MATs that consume the same HOST activations (e.g. the projections of one layer, or a perf sweep): one upload of src1 into the
 * shared device staging buffer args[0].src1, n launches, n downloads into host_dst[i], one synchronisation. */
GGML_B200_API int    ggml_b200_mul_mat_host_batch(const ggml_b200_mul_mat_args * args, int32_t n, const float * host_src1, float * const * host_dst, void * stream);

/* ---------------------------------------------------------------------------------------------
 * Row-sharded MUL_MAT across GPUs (one process per GPU), fused with the exchange: rank r computes rows
 * [row_offset, row_offset + M) of the full product and the mat-vec kernel stores every result directly into each
 * peer's full-length y over NVLink (peer pointers from CUDA IPC), then publishes `epoch` in every peer's flag array;
 * ggml_b200_gather_wait makes the stream wait until all ranks have published.  Replaces the reference's split-buffer
 * gather (cudaMemcpy3DPeerAsync + events, src/ggml-cuda/ggml-cuda.cu:1333-1351, 1621-1647).  n = 1 mat-vec path only.
 * ------------------------------------------------------------------------------------------- */
typedef struct ggml_b200_gather {
    int32_t    world, rank;          /* <= 8 */
    int64_t    row_offset;           /* first row of this rank's shard in the full y */
    uint32_t   epoch;                /* 0: device-managed counter (CUDA-graph replayable), else an explicit increasing value */
    float *    y_peers[8];           /* full-length y of every rank (own entry included) */
    uint32_t * flag_peers[8];        /* flag array (>= world uint32, zero-initialised) of every rank */
} ggml_b200_gather;

GGML_B200_API int ggml_b200_mul_mat_gather(const ggml_b200_mul_mat_args * args, const ggml_b200_gather * gather, void * stream);
/* 1 if ggml_b200_mul_mat_gather can run this shape (pure query) */
GGML_B200_API int ggml_b200_mul_mat_gather_supported(const ggml_b200_mul_mat_args * args);
GGML_B200_API int ggml_b200_gather_wait(const uint32_t * flags_local, int32_t world, uint32_t epoch, void * stream);
/* CUDA-IPC plumbing for the peer buffers: allocate (zeroed) + export a 64-byte handle; open / close a peer's handle */
GGML_B200_API int ggml_b200_ipc_alloc(size_t bytes, void ** dev_ptr, void * handle64);
GGML_B200_API int ggml_b200_ipc_free(void * dev_ptr);
GGML_B200_API int ggml_b200_ipc_open(const void * handle64, void ** dev_ptr);
GGML_B200_API int ggml_b200_ipc_close(void * dev_ptr);

/* ---------------------------------------------------------------------------------------------
 * MUL_MAT_ID (src/ggml.c:2735-2762): as[K, M, n_expert] quantized, b[K, nb1cols, n_tok] f32,
 * ids[n_used, n_tok] i32 (row stride ids_nb1 bytes) -> dst[M, n_used, n_tok] f32 contiguous:
 *   dst[t][e][:] = as[ids[t][e]] . b[t][e % nb1cols]
 * Expert routing is resolved on the device (no host synchronisation).
 * ------------------------------------------------------------------------------------------- */
typedef struct ggml_b200_mul_mat_id_args {
    int32_t      type;
    int32_t      flags;
    int64_t      K, M, n_expert, n_used, nb1cols, n_tok;
    size_t       nb01, nb02;              /* expert matrices: row stride, matrix stride (bytes) */
    size_t       nb11, nb12;              /* b: column stride, token stride (bytes) */
    size_t       ids_nb1;                 /* ids: token stride (bytes) */
    const void * src0;
    const float* src1;
    const int32_t * ids;
    float *      dst;
    void *       workspace;
    size_t       workspace_size;
} ggml_b200_mul_mat_id_args;

GGML_B200_API size_t ggml_b200_mul_mat_id_workspace_size(const ggml_b200_mul_mat_id_args * args);
GGML_B200_API int    ggml_b200_mul_mat_id(const ggml_b200_mul_mat_id_args * args, void * stream);

/* ---------------------------------------------------------------------------------------------
 * Block formats (src/ggml-common.h, src/ggml-quants.c) — bit-exact with the reference's
 * dequantize_row_* / quantize_row_*_ref.
 * ------------------------------------------------------------------------------------------- */
GGML_B200_API size_t ggml_b200_row_size(int32_t type, int64_t k);                 /* = ggml_row_size */
/* dst[n] (f32 or f16 per dst_type) = dequantize(src blocks); n % block size == 0 */
GGML_B200_API int    ggml_b200_dequantize(int32_t type, const void * src, void * dst, int32_t dst_type, int64_t n, void * stream);
/* f32 -> Q8_0 / Q4_0 blocks (quantize_row_q8_0_ref / quantize_row_q4_0_ref), n % 32 == 0 */
GGML_B200_API int    ggml_b200_quantize(int32_t type, const float * src, void * dst, int64_t n, void * stream);
/* activation quantizer exactly as the CPU backend applies it before vec_dot: rows of K f32 -> int8 records
 * (debug/verification entry point; layout: ggml_b200_act_record_size bytes per row: q[K] | bsums int16[K/16] | d f32[]) */
GGML_B200_API size_t ggml_b200_act_record_size(int32_t weight_type, int64_t K);
GGML_B200_API int    ggml_b200_quantize_activations(int32_t weight_type, const float * src, size_t row_stride_bytes,
                                                    int64_t nrows, int64_t K, void * dst_records, void * stream);

/* ---------------------------------------------------------------------------------------------
 * The small ops either side of the mat-mul in the examples/gpt-2 graph (SURVEY.md §8f-1), so that a whole
 * token graph runs on the device.  Tensors are described like ggml tensors: ne[] in elements, nb[] in bytes.
 * Replaces src/ggml-cuda/{getrows,binbcast,norm,scale,diagmask,softmax,unary,cpy,mmv}.cu; semantics follow the
 * CPU backend (src/ggml-cpu/ggml-cpu.c), see ggml_b200/csrc/ops.cu for line references.
 * ------------------------------------------------------------------------------------------- */
typedef struct ggml_b200_tensor {
    void *  data;      /* device */
    int32_t type;      /* enum ggml_type id: 0 f32, 1 f16, 26 i32, or a block-quantized type */
    int64_t ne[4];
    size_t  nb[4];
} ggml_b200_tensor;

enum ggml_b200_unary { GGML_B200_UNARY_GELU = 0, GGML_B200_UNARY_SILU = 1, GGML_B200_UNARY_RELU = 2, GGML_B200_UNARY_TANH = 3,
                       GGML_B200_UNARY_NEG = 4, GGML_B200_UNARY_ABS = 5, GGML_B200_UNARY_GELU_QUICK = 6, GGML_B200_UNARY_SIGMOID = 7,
                       GGML_B200_UNARY_EXP = 8, GGML_B200_UNARY_SQR = 9, GGML_B200_UNARY_SQRT = 10 };

GGML_B200_API int ggml_b200_op_get_rows(const ggml_b200_tensor * src0, const ggml_b200_tensor * ids, const ggml_b200_tensor * dst, void * stream);
/* op: 0 add, 1 mul, 2 sub, 3 div; src1 broadcasts into dst's shape; dst may alias src0 */
GGML_B200_API int ggml_b200_op_bin_bcast(int32_t op, const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, void * stream);
GGML_B200_API int ggml_b200_op_norm(int32_t rms, const ggml_b200_tensor * src, const ggml_b200_tensor * dst, float eps, void * stream);
/* NORM / RMS_NORM followed by MUL(gain[ne0]) and ADD(bias[ne0]) in one pass; the three ggml nodes' outputs are all written */
GGML_B200_API int ggml_b200_op_norm_affine(int32_t rms, const ggml_b200_tensor * src, const ggml_b200_tensor * dst_norm, const float * gain, const ggml_b200_tensor * dst_mul,
                                           const float * bias, const ggml_b200_tensor * dst_add, float eps, void * stream);
GGML_B200_API int ggml_b200_op_scale(const float * src, float * dst, float s, int64_t n, void * stream);
GGML_B200_API int ggml_b200_op_diag_mask_inf(const float * src, float * dst, int64_t ne0, int64_t ne1, int64_t n, int32_t n_past, void * stream);
GGML_B200_API int ggml_b200_op_unary(int32_t uop, const float * src, float * dst, int64_t n, void * stream);
GGML_B200_API int ggml_b200_op_soft_max(const float * src, const void * mask, int32_t mask_type, float * dst, int64_t ne0, int64_t ne1, int64_t ne2, int64_t ne3,
                                        float scale, float max_bias, void * stream);
/* SCALE -> DIAG_MASK_INF(n_past) -> SOFT_MAX in one row pass: softmax over x * scale with element i0 of row i1 masked where i0 > diag_n_past + i1
 * (diag_n_past < 0: no mask; then identical to ggml_b200_op_soft_max) */
GGML_B200_API int ggml_b200_op_soft_max_diag(const float * src, const void * mask, int32_t mask_type, float * dst, int64_t ne0, int64_t ne1, int64_t ne2, int64_t ne3,
                                             float scale, float max_bias, int32_t diag_n_past, void * stream);
GGML_B200_API int ggml_b200_op_cpy(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream);
/* two independent float copies of the same element count in one launch (the K and V cache updates of a layer) */
GGML_B200_API int ggml_b200_op_cpy2(const ggml_b200_tensor * src_a, const ggml_b200_tensor * dst_a, const ggml_b200_tensor * src_b, const ggml_b200_tensor * dst_b, void * stream);
/* GGML_OP_FLASH_ATTN_EXT (include/ggml.h:1785-1800): q f32 [d, n_q, n_head, b], k / v [d, n_kv, n_head_kv, b] in f16, f32 or any block format this
 * library decodes (quantized KV caches), mask f16 [n_kv, >= n_q] or NULL -> dst f32 [d, n_head, n_q, b]; d <= 256.  Replaces src/ggml-cuda/fattn*.cu. */
GGML_B200_API int ggml_b200_op_flash_attn_ext(const ggml_b200_tensor * q, const ggml_b200_tensor * k, const ggml_b200_tensor * v, const ggml_b200_tensor * mask,
                                              const ggml_b200_tensor * dst, float scale, float max_bias, float logit_softcap, void * stream);
/* float mat-mul: src0 f32/f16 [K, M, ne02, ne03] (any strides) x src1 f32 [K, N, ne12, ne13] -> dst f32 */
GGML_B200_API int ggml_b200_op_mul_mat_f(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, void * stream);

/* ---------------------------------------------------------------------------------------------
 * Introspection
 * ------------------------------------------------------------------------------------------- */
GGML_B200_API const char * ggml_b200_last_error(void);
GGML_B200_API int          ggml_b200_device_count(void);
GGML_B200_API int          ggml_b200_sm_count(void);
/* one-time per-device setup (control block of the mat-vec scheduler and the split-K flags) for the CURRENT device.  Launches do it
 * lazily; call it explicitly before the first launch that falls inside a stream capture (allocation is not capturable). */
GGML_B200_API int          ggml_b200_prepare(void);
/* number of kernels this library has launched since load (for bench.py's gpu_launches) */
GGML_B200_API uint64_t     ggml_b200_launch_count(void);
/* developer diagnostic kept for ABI stability: the GEMM kernel records no per-CTA stamps, so this copies nothing and returns 0 */
GGML_B200_API int          ggml_b200_debug_gemm_trace(uint64_t * host_dst, int32_t max_ctas);
GGML_B200_API const char * ggml_b200_version(void);
/* developer aid (GGML_B200_SB_DEBUG=1): %globaltimer stamps of CTA 0 for the last 32 mat-vec launches, 8 per launch */
GGML_B200_API int          ggml_b200_debug_trace(unsigned long long * out256);

#ifdef __cplusplus
}
#endif
#endif /* GGML_B200_H */
