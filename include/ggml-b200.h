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
    /* indices and positions of the small ops (ggml_b200_tensor) */
    GGML_B200_TYPE_I32 = 26,
    /* the 2-byte element types GGML_OP_REPEAT moves besides f16 */
    GGML_B200_TYPE_I16 = 25, GGML_B200_TYPE_BF16 = 30,
    /* GGML_OP_COUNT_EQUAL's scalar result */
    GGML_B200_TYPE_I64 = 27,
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
/* dense fp16 [M][K] (row stride nb01 bytes) x fp16 [N][K] (row stride nb11 bytes) -> f32 [N][M] on the tensor cores: both operands go
   straight into the GEMM by TMA, with no conversion pass.  This is GGML_OP_MUL_MAT with f16 src0 and f16 src1, the product ggml_conv_1d /
   ggml_conv_2d build (w: the IM2COL result, x: the conv kernel).  Eligible: N >= 9, K % 64 == 0, both row strides multiples of 16 bytes.
   workspace_size = 0 from the size function: shape not eligible. */
GGML_B200_API size_t ggml_b200_mul_mat_f16_f16_workspace_size(int64_t M, int64_t N, int64_t K);
GGML_B200_API int    ggml_b200_mul_mat_f16_f16(const void * w, size_t nb01, const void * x, size_t nb11, float * y, int64_t M, int64_t N, int64_t K,
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
 * Expert routing is resolved on the device (no host synchronisation).  An id outside [0, n_expert) (the CPU backend asserts on
 * it) gives dst[t][e][:] = 0, on the per-pair and on the expert-grouped form alike; no weight row is read for it.
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
    int32_t type;      /* enum ggml_b200_type: f32, f16, i32 or a block-quantized type */
    int64_t ne[4];
    size_t  nb[4];
} ggml_b200_tensor;

enum ggml_b200_unary { GGML_B200_UNARY_GELU = 0, GGML_B200_UNARY_SILU = 1, GGML_B200_UNARY_RELU = 2, GGML_B200_UNARY_TANH = 3,
                       GGML_B200_UNARY_NEG = 4, GGML_B200_UNARY_ABS = 5, GGML_B200_UNARY_GELU_QUICK = 6, GGML_B200_UNARY_SIGMOID = 7,
                       GGML_B200_UNARY_EXP = 8, GGML_B200_UNARY_SQR = 9, GGML_B200_UNARY_SQRT = 10,
                       /* GGML_OP_SIN / GGML_OP_COS: sinf / cosf (within 2 ulp, not the fast intrinsics) */
                       GGML_B200_UNARY_SIN = 11, GGML_B200_UNARY_COS = 12,
                       /* GGML_UNARY_OP_STEP: x > 0 ? 1 : 0 (NaN gives 0); the gradient of RELU */
                       GGML_B200_UNARY_STEP = 13 };

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
/* float mat-mul: src0 f32/f16 [K, M, ne02, ne03] (any strides) x src1 f32 [K, N, ne12, ne13] -> dst f32; src1 may also be f16 when src0
 * is f16 (read as is: the CPU backend rounds an f32 src1 to f16 for an f16 src0, and takes an f16 src1 unchanged) */
GGML_B200_API int ggml_b200_op_mul_mat_f(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_ROPE, forward (ggml_rope_ext / ggml_rope_multi): src f32 or f16 [ne0, n_head, n_pos, b] -> dst of the same type and shape (any row
 * strides, dim 0 contiguous; dst may be src itself).  pos i32 [n_pos] (MROPE / VISION: [4 * n_pos]) is read on the device.  freq_factors: NULL or
 * f32 [>= n_dims/2] (VISION: >= n_dims).  The per-op constants are computed by the caller with the CPU backend's expressions:
 * theta_scale = powf(freq_base, -2.0f/n_dims), corr_dims from ggml_rope_yarn_corr_dims, and mscale = attn_factor, multiplied by
 * (1 + 0.1 logf(1/freq_scale)) when ext_factor != 0. */
typedef struct ggml_b200_rope_params {
    int32_t n_dims;        /* rotated dimensions: even, <= ne0 (VISION: == ne0/2), <= 1024 */
    int32_t mode;          /* 0 normal (adjacent pairs), 2 NEOX (i, i + n_dims/2), 8 MROPE, 24 VISION (i, i + n_dims) */
    int32_t sections[4];   /* MROPE / VISION: dimensions per position stream, not all zero */
    float   freq_scale;
    float   ext_factor;
    float   mscale;
    float   theta_scale;
    float   corr_dims[2];
} ggml_b200_rope_params;
GGML_B200_API int ggml_b200_op_rope(const ggml_b200_tensor * src, const ggml_b200_tensor * pos, const ggml_b200_tensor * freq_factors, const ggml_b200_tensor * dst,
                                    const ggml_b200_rope_params * params, void * stream);
/* GGML_OP_ARGSORT: src f32 [ne0, ne1, ne2, ne3] (any row strides, dim 0 contiguous), 1 <= ne0 <= 1024 -> dst i32 of the same shape, contiguous:
 * per row the indices that order it ascending (order 0) or descending (order 1).  Ties come out in ascending index, -0.0 equals +0.0 and
 * NaNs sort after every number in both orders, so each row of dst is a permutation of 0 .. ne0-1.  No allocation, no host sync. */
GGML_B200_API int ggml_b200_op_argsort(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t order, void * stream);
/* GGML_OP_SUM_ROWS: src f32 [ne0, ne1, ne2, ne3] (any row strides, dim 0 contiguous) -> dst f32 [1, ne1, ne2, ne3] (any strides); each row
 * is accumulated in double and rounded once, as the CPU backend does. */
GGML_B200_API int ggml_b200_op_sum_rows(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_CONCAT: src0 and src1 both f32 or both i32 (src0 contiguous along dim 0, src1 any strides) -> dst of the same type (any strides),
 * src1 appended after src0 along dim (0 .. 3; any other value: GGML_B200_EINVAL).  Outside dim the three shapes agree.  Copies 4-byte
 * words, so the result is bit-identical. */
GGML_B200_API int ggml_b200_op_concat(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, int32_t dim, void * stream);
/* GGML_OP_SSM_CONV: sx f32 [d_conv - 1 + n_t, d_inner, n_s] (packed rows: nb1 == ne0 * 4; any nb2), c f32 [d_conv, d_inner] (packed rows too:
 * the CPU backend reads row i1 of c at i1 * d_conv whatever its nb1)
 * -> dst f32 [d_inner, n_t, n_s] (dim 0 contiguous): dst[i1, t, s] = sum_{i0 < d_conv} sx[t + i0, i1, s] * c[i0, i1], each product and sum
 * rounded separately in ascending i0, bit-identical to the CPU backend. */
GGML_B200_API int ggml_b200_op_ssm_conv(const ggml_b200_tensor * sx, const ggml_b200_tensor * c, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_SSM_SCAN (Mamba-1): s f32 [d_state, d_inner, n_s], x and dt f32 [d_inner, n_t, n_s], A f32 [d_state, d_inner] (all four contiguous),
 * B and C f32 [d_state, n_t, n_s] (dim 0 contiguous, any nb1 / nb2: views of x_db) -> dst f32, contiguous, ne(x) + ne(s) elements: y in x's
 * layout, then from byte offset x.nb[3] the final states in s's layout.  Per row and sequence, token by token:
 * dt' = softplus(dt) (dt above 20 kept), state = state * exp(dt' A) + B (x dt'), y = sum over d_state of state * C, in the CPU backend's
 * order and rounding; any d_state (the states are kept in dst, not in registers), n_s <= 65535. */
GGML_B200_API int ggml_b200_op_ssm_scan(const ggml_b200_tensor * s, const ggml_b200_tensor * x, const ggml_b200_tensor * dt, const ggml_b200_tensor * A,
                                        const ggml_b200_tensor * B, const ggml_b200_tensor * C, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_RWKV_WKV6 (the RWKV-6 time-mix recurrence): k, v, r, td f32 [S, H, T], tf f32 with S * H values, s f32 with S * S * H * n_seqs values
 * (n_seqs = s->ne[1]), all contiguous -> dst f32 [S * H, T + S * n_seqs], contiguous: y [S * H, T], then the final states in s's layout.
 * Sequence q owns tokens [q T / n_seqs, (q + 1) T / n_seqs) (T % n_seqs == 0, else GGML_B200_EINVAL) and starts from its state in s.  Per
 * token, head and state element (i, j): kv = v[j] k[i]; y[j] += (kv tf[i] + state[i][j]) r[i], summed in ascending i; state[i][j] =
 * state[i][j] td[i] + kv, rounded as the CPU backend's vector path.  S <= 256.  T == 0 writes nothing. */
GGML_B200_API int ggml_b200_op_rwkv_wkv6(const ggml_b200_tensor * k, const ggml_b200_tensor * v, const ggml_b200_tensor * r, const ggml_b200_tensor * tf,
                                         const ggml_b200_tensor * td, const ggml_b200_tensor * s, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_GATED_LINEAR_ATTN: as ggml_b200_op_rwkv_wkv6 with q and g in place of r and td and no tf: temp = state[i][j] g[i] + kv;
 * y[j] += temp (q[i] scale); state[i][j] = temp. */
GGML_B200_API int ggml_b200_op_gated_linear_attn(const ggml_b200_tensor * k, const ggml_b200_tensor * v, const ggml_b200_tensor * q, const ggml_b200_tensor * g,
                                                 const ggml_b200_tensor * s, const ggml_b200_tensor * dst, float scale, void * stream);
/* GGML_OP_IM2COL (ggml_im2col; the first node of ggml_conv_1d / ggml_conv_2d): the op_params of the node, in their order */
typedef struct ggml_b200_im2col_params {
    int32_t s0, s1;        /* stride along the width / height, >= 1 (s1, p1, d1: 2-D only) */
    int32_t p0, p1;        /* padding (zeros) */
    int32_t d0, d1;        /* dilation, >= 1 */
    int32_t is_2D;         /* 0: 1-D, 1: 2-D */
} ggml_b200_im2col_params;
/* src0: the conv kernel (only its extents are read: KW = ne0, 2-D KH = ne1), src1: the input f32 [IW, IC, N, 1] (1-D) or [IW, IH, IC, N] (2-D),
 * contiguous along dim 0 -> dst f32 or f16, packed, [IC KW, OW, N, 1] (1-D) or [IC KH KW, OW, OH, N] (2-D), OW and OH the output sizes
 * (in + 2 p - d (k - 1) - 1) / s + 1; an f16 dst needs an f16 src0, as the CPU backend asserts.  Bit-identical to the CPU backend in both dst
 * types; a channel's rows are read as packed, as the CPU backend reads them.  src1 offsets of an image / a channel beyond INT32_MAX bytes:
 * GGML_B200_EUNSUPPORTED (the CPU backend keeps them in an int). */
GGML_B200_API int ggml_b200_op_im2col(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst,
                                      const ggml_b200_im2col_params * params, void * stream);
/* GGML_OP_POOL_2D (ggml_pool_2d): the op_params of the node, in their order */
typedef struct ggml_b200_pool_params {
    int32_t op;            /* 0 MAX, 1 AVG (2, COUNT: GGML_B200_EINVAL, as the CPU backend aborts on it) */
    int32_t k0, k1;        /* window width / height, >= 1 */
    int32_t s0, s1;        /* stride, >= 1 */
    int32_t p0, p1;        /* padding, as stored in op_params: ggml_pool_2d's float paddings truncated */
} ggml_b200_pool_params;
/* src f32 [IW, IH, C, N] (elements packed along dim 0, any row / channel / image strides) -> dst f32 [OW, OH, C, N], packed.  OW and OH are
 * dst's own extents: ggml_pool_2d computes them from its float paddings, so they are never re-derived here.  Window (ox, oy) starts at
 * (ox s0 - p0, oy s1 - p1); taps outside the input are skipped.  MAX starts at -FLT_MAX and takes a tap only when it is greater (NaN taps are
 * ignored, a window of padding or NaN gives -FLT_MAX); AVG sums the in-range taps in row order and divides by k0 k1.  Bit-identical to the
 * CPU backend.  dst C or N different from src's: GGML_B200_EINVAL. */
GGML_B200_API int ggml_b200_op_pool_2d(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, const ggml_b200_pool_params * params, void * stream);
/* GGML_OP_UPSCALE (nearest; ggml_upscale / ggml_upscale_ext): src f32 (any strides) -> dst f32 (any strides), dst extents >= src's (else
 * GGML_B200_EINVAL).  dst (i0, i1, i2, i3) = src (i0 / sf0, ...) truncated, sf_i = (float) dst ne_i / src ne_i, computed here from the two
 * descriptors in float as the CPU backend computes them: bit-identical. */
GGML_B200_API int ggml_b200_op_upscale(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_LEAKY_RELU: src and dst f32 of the same shape (else GGML_B200_EINVAL), both contiguous along dim 0, any other strides; dst may be
 * src itself (in place).  dst = ((x > 0) ? x : 0) + slope ((x < 0) ? x : 0), each step rounded as the CPU backend rounds it: NaN and -0 give
 * +0.  Bit-identical. */
GGML_B200_API int ggml_b200_op_leaky_relu(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, float slope, void * stream);
/* GGML_OP_REPEAT: src and dst of one type with 4-byte (f32, i32) or 2-byte (f16, bf16, i16) elements, both contiguous along dim 0, any other
 * strides; every dst extent a whole multiple of src's (else GGML_B200_EINVAL).  dst (i0, i1, i2, i3) = src (i0 % ne00, i1 % ne01, ...), moved
 * as raw words: every bit pattern (NaN payloads included) is kept. */
GGML_B200_API int ggml_b200_op_repeat(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_WIN_PART (ggml_win_part): src f32 [C, W0, H0, 1] -> dst f32 [C, w, w, npx npy], both packed; npx, npy, w the node's op_params.
 * Window py npx + px holds the image pixels (px w + i1, py w + i2), zeros where it runs past the image.  Raw 4-byte words: bit-identical
 * (NaN payloads and -0 kept).  npx != ceil(W0 / w), npy != ceil(H0 / w), w < 1 or dst extents that disagree: GGML_B200_EINVAL. */
GGML_B200_API int ggml_b200_op_win_part(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t npx, int32_t npy, int32_t w, void * stream);
/* GGML_OP_WIN_UNPART (ggml_win_unpart): src f32 [C, w, w, np] -> dst f32 [C, W0, H0, 1], both packed; the inverse of WIN_PART, dropping the
 * padding.  Raw words: bit-identical.  np < ceil(W0 / w) ceil(H0 / w) (the reads would leave src), w < 1: GGML_B200_EINVAL. */
GGML_B200_API int ggml_b200_op_win_unpart(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t w, void * stream);
/* GGML_OP_GET_REL_POS (ggml_get_rel_pos): src f16 [C, 2w - 1] -> dst f16 [C, w, w], both packed: dst[i2, i1, :] = src[(w - 1 - i1) + i2, :],
 * raw 2-byte words (bit-identical).  Other types (BF16 included): GGML_B200_EUNSUPPORTED. */
GGML_B200_API int ggml_b200_op_get_rel_pos(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_ADD_REL_POS (ggml_add_rel_pos[_inplace]): src0 f32 [L L, A B, P, 1], pw and ph f32 [L, A, B, P], dst like src0, all packed; dst may
 * be src0 (in place).  dst[r, kh L + kw] = src0[r, kh L + kw] + ph[r, kh] + pw[r, kw], the two adds in the CPU backend's order (ph first when
 * kh <= kw, pw first otherwise): bit-identical.  src0 with ne3 > 1: GGML_B200_EUNSUPPORTED; extents that disagree: GGML_B200_EINVAL. */
GGML_B200_API int ggml_b200_op_add_rel_pos(const ggml_b200_tensor * src0, const ggml_b200_tensor * pw, const ggml_b200_tensor * ph, const ggml_b200_tensor * dst,
                                           void * stream);
/* GGML_OP_CONV_TRANSPOSE_2D (ggml_conv_transpose_2d_p0): kernel f16 [Kw, Kh, Cout, Cin] (Kw x Kh planes packed), input f32 [W, H, Cin, 1]
 * (contiguous along dim 0) -> dst f32 [(W-1) s + Kw, (H-1) s + Kh, Cout, 1] packed, padding 0.  The input is rounded to fp16 (to nearest even,
 * as the CPU backend rounds it); each tap's dot over Cin is an f32 sum of exact fp16 x fp16 products; the taps are added from +0.0 in the CPU
 * backend's order (ascending input row, then column).  Only the order inside a dot differs from the CPU backend.  A batch (ne3 > 1):
 * GGML_B200_EUNSUPPORTED; stride < 1 or extents that disagree: GGML_B200_EINVAL. */
GGML_B200_API int ggml_b200_op_conv_transpose_2d(const ggml_b200_tensor * kernel, const ggml_b200_tensor * input, const ggml_b200_tensor * dst,
                                                 int32_t stride, void * stream);

/* The ops ggml_opt's backward and optimizer graphs add (ggml_build_backward_expand, ggml_opt_step_adamw), all f32 unless stated.
 * GGML_OP_OUT_PROD (the gradient of MUL_MAT): src0 [ne0, K, ne02, ne03] contiguous along dim 0, src1 [ne1, K, ne2, ne3] with any strides
 * (ggml_transpose(grad) is the common case) -> dst [ne0, ne1, ne2, ne3] packed; ne2 % ne02 == 0 and ne3 % ne03 == 0 (broadcast as MUL_MAT).
 * dst[i0, i1] = sum over k of src0[i0, k] src1[i1, k], one fused multiply-add per term in ascending k from +0: the CPU backend's chain on
 * the elements of its SIMD body (i0 below ne0 rounded down to 32), within NMSE 1e-12 elsewhere.  K = 0 gives zeros.  f16 or quantized
 * src0: GGML_B200_EUNSUPPORTED. */
GGML_B200_API int ggml_b200_op_out_prod(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_CROSS_ENTROPY_LOSS: logits and labels of one shape, rows contiguous along dim 0 -> dst, a scalar:
 * -1/nr sum over rows and i of labels_i (x_i - max - log sum_j exp(x_j - max)), with the CPU backend's per-row rounding.  The rows are
 * reduced in one fixed order (no atomics): passes repeat bit for bit. */
GGML_B200_API int ggml_b200_op_cross_entropy_loss(const ggml_b200_tensor * logits, const ggml_b200_tensor * labels, const ggml_b200_tensor * dst,
                                                  void * stream);
/* GGML_OP_CROSS_ENTROPY_LOSS_BACK: grad a scalar (read on the device), logits, labels and dst of one shape, all packed:
 * dst = (softmax(logits) - labels) grad[0] / nr, row by row. */
GGML_B200_API int ggml_b200_op_cross_entropy_loss_back(const ggml_b200_tensor * grad, const ggml_b200_tensor * logits, const ggml_b200_tensor * labels,
                                                       const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_OPT_STEP_ADAMW, in place: w (the node's dst, a view of the weight), its gradient g and moments m and v, all of one shape and
 * packed; params f32 [7] = alpha, beta1, beta2, eps, wd, beta1h, beta2h, read on the device by every launch (a replayed CUDA graph sees
 * the values of the step it replays).  w, m and v are updated with the CPU backend's expressions in its order: bit-identical. */
GGML_B200_API int ggml_b200_op_opt_step_adamw(const ggml_b200_tensor * w, const ggml_b200_tensor * g, const ggml_b200_tensor * m, const ggml_b200_tensor * v,
                                              const ggml_b200_tensor * params, void * stream);
/* GGML_OP_ARGMAX: src [ne0, ne1] (rows contiguous along dim 0) -> dst i32 [ne1] (dim 0 contiguous): the CPU backend's rule (the last index
 * of the maximum; a NaN restarts the search after it; a trailing run of NaNs is ignored; all NaN gives 0).  Exact. */
GGML_B200_API int ggml_b200_op_argmax(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_COUNT_EQUAL: src0 and src1 i32 of one shape [ne0, ne1, 1, 1] (any strides) -> dst i64 scalar, the number of equal pairs.  Exact.
 * ne2 or ne3 > 1: GGML_B200_EUNSUPPORTED (the CPU backend's row walk reads other rows then). */
GGML_B200_API int ggml_b200_op_count_equal(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_SUM: src (contiguous along dim 0, any other strides) -> dst a scalar: the sum in double, rounded once, in one fixed order. */
GGML_B200_API int ggml_b200_op_sum(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream);
/* GGML_OP_REPEAT_BACK: src -> dst, both contiguous along dim 0 (any other strides), every src extent a whole multiple of dst's:
 * dst (k) = the sum over the repeats of src into dst's shape, added in the CPU backend's loop order: bit-identical.  Other types than f32:
 * GGML_B200_EUNSUPPORTED. */
GGML_B200_API int ggml_b200_op_repeat_back(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream);

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
GGML_B200_API const char * ggml_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* GGML_B200_H */
