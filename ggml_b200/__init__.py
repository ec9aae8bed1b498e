"""ggml_b200 — H100-native (sm_90a) kernels for ggml's block-quantized MUL_MAT / MUL_MAT_ID hot path.

The product is native code: `libggml-b200-kernels.so` (hand-written CUDA behind the C ABI of
include/ggml-b200.h) and `libggml-b200.so` (the ggml backend plug-in built on it).  This Python module is only
a ctypes mirror of that C ABI for tests and benchmarks; PyTorch supplies device memory and streams.
There is no CPU fallback: importing works anywhere, but every compute entry point raises if the CUDA library
is missing or reports an error.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

PKG = Path(__file__).resolve().parent
KERNELS_SO = PKG / "libggml-b200-kernels.so"
BACKEND_SO = PKG / "libggml-b200.so"

# enum ggml_type ids (reference include/ggml.h:351-390)
F32, F16, Q4_0, Q8_0, Q4_K, Q5_K, Q6_K = 0, 1, 2, 8, 12, 13, 14
Q4_1, Q5_0, Q5_1, Q2_K, Q3_K, IQ4_NL, IQ4_XS = 3, 6, 7, 10, 11, 20, 23      # SURVEY §8f-2 formats
IQ2_XXS, IQ3_XXS, IQ1_S = 16, 18, 19                                       # grid-codebook i-quants (generic kernels)
IQ2_XS, IQ3_S, IQ2_S, IQ1_M, TQ1_0, TQ2_0 = 17, 21, 22, 29, 34, 35
QUANT_TYPES = (Q4_0, Q8_0, Q4_K, Q5_K, Q6_K)
NEXT_TYPES = (Q4_1, Q5_0, Q5_1, Q2_K, Q3_K, IQ4_NL, IQ4_XS)
TYPE_NAMES = {F32: "f32", F16: "f16", Q4_0: "q4_0", Q8_0: "q8_0", Q4_K: "q4_K", Q5_K: "q5_K", Q6_K: "q6_K",
              Q4_1: "q4_1", Q5_0: "q5_0", Q5_1: "q5_1", Q2_K: "q2_K", Q3_K: "q3_K", IQ4_NL: "iq4_nl", IQ4_XS: "iq4_xs",
              IQ2_XXS: "iq2_xxs", IQ3_XXS: "iq3_xxs", IQ1_S: "iq1_s",
              IQ2_XS: "iq2_xs", IQ3_S: "iq3_s", IQ2_S: "iq2_s", IQ1_M: "iq1_m", TQ1_0: "tq1_0", TQ2_0: "tq2_0"}

MM_AUTO, MM_GENERIC, MM_GEMV, MM_GEMM, MM_GEMV_V1, MM_SRC0_STATIC, MM_SRC1_STATIC = 0, 1, 2, 4, 8, 16, 32
MM_GEMV_MMA, MM_GEMV_DP4A = 64, 128


class B200Error(RuntimeError):
    pass


class MulMatArgs(C.Structure):
    _fields_ = [("type", C.c_int32), ("flags", C.c_int32),
                ("K", C.c_int64), ("M", C.c_int64), ("N", C.c_int64),
                ("ne02", C.c_int64), ("ne03", C.c_int64), ("ne12", C.c_int64), ("ne13", C.c_int64),
                ("nb01", C.c_size_t), ("nb02", C.c_size_t), ("nb03", C.c_size_t),
                ("nb11", C.c_size_t), ("nb12", C.c_size_t), ("nb13", C.c_size_t),
                ("src0", C.c_void_p), ("src1", C.c_void_p), ("dst", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_size", C.c_size_t)]


class MulMatIdArgs(C.Structure):
    _fields_ = [("type", C.c_int32), ("flags", C.c_int32),
                ("K", C.c_int64), ("M", C.c_int64), ("n_expert", C.c_int64), ("n_used", C.c_int64),
                ("nb1cols", C.c_int64), ("n_tok", C.c_int64),
                ("nb01", C.c_size_t), ("nb02", C.c_size_t), ("nb11", C.c_size_t), ("nb12", C.c_size_t),
                ("ids_nb1", C.c_size_t),
                ("src0", C.c_void_p), ("src1", C.c_void_p), ("ids", C.c_void_p), ("dst", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_size", C.c_size_t)]


_lib = None


def lib() -> C.CDLL:
    """The kernel-launch shim.  Fails loudly when it has not been built (no fallback)."""
    global _lib
    if _lib is None:
        if not KERNELS_SO.exists():
            raise B200Error(f"{KERNELS_SO} is not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(str(KERNELS_SO))
        L.ggml_b200_last_error.restype = C.c_char_p
        L.ggml_b200_version.restype = C.c_char_p
        L.ggml_b200_launch_count.restype = C.c_uint64
        L.ggml_b200_row_size.restype = C.c_size_t
        L.ggml_b200_row_size.argtypes = [C.c_int32, C.c_int64]
        L.ggml_b200_act_record_size.restype = C.c_size_t
        L.ggml_b200_act_record_size.argtypes = [C.c_int32, C.c_int64]
        L.ggml_b200_quantize_activations.argtypes = [C.c_int32, C.c_void_p, C.c_size_t, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]
        L.ggml_b200_mul_mat_workspace_size.restype = C.c_size_t
        L.ggml_b200_mul_mat_workspace_size.argtypes = [C.POINTER(MulMatArgs)]
        L.ggml_b200_mul_mat_plan.argtypes = [C.POINTER(MulMatArgs)]
        L.ggml_b200_mul_mat.argtypes = [C.POINTER(MulMatArgs), C.c_void_p]
        L.ggml_b200_mul_mat_host.argtypes = [C.POINTER(MulMatArgs), C.c_void_p, C.c_void_p, C.c_void_p]
        L.ggml_b200_mul_mat_id_workspace_size.restype = C.c_size_t
        L.ggml_b200_mul_mat_id_workspace_size.argtypes = [C.POINTER(MulMatIdArgs)]
        L.ggml_b200_mul_mat_id.argtypes = [C.POINTER(MulMatIdArgs), C.c_void_p]
        L.ggml_b200_dequantize.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p]
        L.ggml_b200_quantize.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        _lib = L
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise B200Error(f"{what} failed ({rc}): {lib().ggml_b200_last_error().decode()}")


def row_size(t: int, k: int) -> int:
    return int(lib().ggml_b200_row_size(t, k))


def launch_count() -> int:
    return int(lib().ggml_b200_launch_count())


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Workspace:
    """Grow-only device scratch (a torch uint8 tensor) handed to the C ABI."""

    def __init__(self):
        self.t = None

    def get(self, nbytes: int):
        import torch
        if self.t is None or self.t.numel() < nbytes:
            self.t = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device="cuda")
        return self.t


_ws = Workspace()


def mul_mat_args(t, W, X, Y, M, N, K, batch=(1, 1, 1, 1), flags=MM_AUTO, nb=None, workspace=None) -> MulMatArgs:
    """W: cuda uint8 tensor of packed blocks; X: cuda float32; Y: cuda float32 [ne13, ne12, N, M].  workspace: a cuda uint8 tensor
    handed over whole (its size is what the launch may use), None for the shared grow-only one."""
    ne02, ne03, ne12, ne13 = batch
    rb = row_size(t, K)
    a = MulMatArgs()
    a.type, a.flags, a.K, a.M, a.N = t, flags, K, M, N
    a.ne02, a.ne03, a.ne12, a.ne13 = ne02, ne03, ne12, ne13
    if nb is None:
        a.nb01, a.nb02, a.nb03 = rb, rb * M, rb * M * ne02
        a.nb11, a.nb12, a.nb13 = K * 4, K * 4 * N, K * 4 * N * ne12
    else:
        a.nb01, a.nb02, a.nb03, a.nb11, a.nb12, a.nb13 = nb
    a.src0, a.src1, a.dst = W.data_ptr(), X.data_ptr(), Y.data_ptr()
    ws = workspace if workspace is not None else _ws.get(int(lib().ggml_b200_mul_mat_workspace_size(C.byref(a))))
    a.workspace, a.workspace_size = ws.data_ptr(), ws.numel()
    return a


def mul_mat(t, W, X, M, N, K, batch=(1, 1, 1, 1), flags=MM_AUTO, out=None, nb=None, workspace=None):
    """GGML_OP_MUL_MAT on the current CUDA stream.  Returns Y[ne13, ne12, N, M] (float32, cuda)."""
    import torch
    ne02, ne03, ne12, ne13 = batch
    Y = out if out is not None else torch.empty((ne13, ne12, N, M), dtype=torch.float32, device="cuda")
    a = mul_mat_args(t, W, X, Y, M, N, K, batch, flags, nb, workspace)
    check(lib().ggml_b200_mul_mat(C.byref(a), _stream()), "ggml_b200_mul_mat")
    return Y


def mul_mat_plan(t, M, N, K, flags=MM_AUTO) -> int:
    import torch
    a = MulMatArgs()
    a.type, a.flags, a.K, a.M, a.N = t, flags, K, M, N
    a.ne02 = a.ne03 = a.ne12 = a.ne13 = 1
    rb = row_size(t, K)
    a.nb01, a.nb02, a.nb03, a.nb11, a.nb12, a.nb13 = rb, rb * M, rb * M, K * 4, K * 4 * N, K * 4 * N
    a.src0 = a.src1 = a.dst = 256      # aligned dummies: plan() never dereferences
    return int(lib().ggml_b200_mul_mat_plan(C.byref(a)))


def mul_mat_id(t, W, X, ids, M, K, n_expert, n_used, nb1cols, n_tok, out=None, workspace=None):
    """GGML_OP_MUL_MAT_ID.  W: packed [n_expert, M, row]; X: f32 [n_tok, nb1cols, K]; ids: int32 [n_tok, >= n_used] (any row stride).
    out: None (a new tensor) or a contiguous f32 [n_tok, n_used, M]; workspace: as for mul_mat."""
    import torch
    Y = out if out is not None else torch.empty((n_tok, n_used, M), dtype=torch.float32, device="cuda")
    rb = row_size(t, K)
    a = MulMatIdArgs()
    a.type, a.flags, a.K, a.M = t, 0, K, M
    a.n_expert, a.n_used, a.nb1cols, a.n_tok = n_expert, n_used, nb1cols, n_tok
    a.nb01, a.nb02, a.nb11, a.nb12 = rb, rb * M, K * 4, K * 4 * nb1cols
    a.ids_nb1 = ids.stride(0) * 4
    a.src0, a.src1, a.ids, a.dst = W.data_ptr(), X.data_ptr(), ids.data_ptr(), Y.data_ptr()
    ws = workspace if workspace is not None else _ws.get(int(lib().ggml_b200_mul_mat_id_workspace_size(C.byref(a))))
    a.workspace, a.workspace_size = ws.data_ptr(), ws.numel()
    check(lib().ggml_b200_mul_mat_id(C.byref(a), _stream()), "ggml_b200_mul_mat_id")
    return Y


def dequantize(t, blocks, n, dtype=None):
    import torch
    dtype = dtype or torch.float32
    out = torch.empty(n, dtype=dtype, device="cuda")
    check(lib().ggml_b200_dequantize(t, blocks.data_ptr(), out.data_ptr(), F32 if dtype == torch.float32 else F16, n, _stream()),
          "ggml_b200_dequantize")
    return out


def quantize(t, x):
    import torch
    x = x.contiguous()
    out = torch.empty(row_size(t, x.numel()), dtype=torch.uint8, device="cuda")
    check(lib().ggml_b200_quantize(t, x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "ggml_b200_quantize")
    return out


def quantize_activations(weight_type, x):
    """x: f32 cuda [rows, K] -> uint8 [rows, record_size] (q | bsums | d), as the mat-vec kernels consume it."""
    import torch
    rows, K = x.shape
    rs = int(lib().ggml_b200_act_record_size(weight_type, K))
    out = torch.zeros((rows, rs), dtype=torch.uint8, device="cuda")
    check(lib().ggml_b200_quantize_activations(weight_type, x.data_ptr(), x.stride(0) * 4, rows, K, out.data_ptr(), _stream()),
          "ggml_b200_quantize_activations")
    return out


# ---------------------------------------------------------------------------------------------------------------
# Row-sharded multi-GPU mat-vec with the exchange fused into the kernel (peer stores over NVLink, CUDA IPC buffers)
class Gather(C.Structure):
    _fields_ = [("world", C.c_int32), ("rank", C.c_int32), ("row_offset", C.c_int64), ("epoch", C.c_uint32),
                ("y_peers", C.c_void_p * 8), ("flag_peers", C.c_void_p * 8)]


class PeerExchange:
    """Per-rank gathered-y buffers (`slots` full-length vectors) + flag array, visible to every peer through CUDA IPC."""

    def __init__(self, m_total: int, rank: int, world: int, row_offset: int, slots: int = 1):
        import torch.distributed as dist
        L = lib()
        L.ggml_b200_ipc_alloc.argtypes = [C.c_size_t, C.POINTER(C.c_void_p), C.c_void_p]
        L.ggml_b200_ipc_open.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.ggml_b200_ipc_close.argtypes = [C.c_void_p]
        L.ggml_b200_ipc_free.argtypes = [C.c_void_p]
        L.ggml_b200_mul_mat_gather.argtypes = [C.POINTER(MulMatArgs), C.POINTER(Gather), C.c_void_p]
        L.ggml_b200_gather_wait.argtypes = [C.c_void_p, C.c_int32, C.c_uint32, C.c_void_p]
        assert 1 <= world <= 8
        self.rank, self.world, self.m_total, self.slots = rank, world, m_total, slots
        self.y_ptr, self.f_ptr = C.c_void_p(), C.c_void_p()
        hy, hf = C.create_string_buffer(64), C.create_string_buffer(64)
        check(L.ggml_b200_ipc_alloc(slots * m_total * 4, C.byref(self.y_ptr), hy), "ipc_alloc(y)")
        check(L.ggml_b200_ipc_alloc(256, C.byref(self.f_ptr), hf), "ipc_alloc(flags)")
        handles = [None] * world
        dist.all_gather_object(handles, (hy.raw, hf.raw))
        self._opened = []
        ys, fs = [], []
        for q, (hyq, hfq) in enumerate(handles):
            if q == rank:
                py, pf = self.y_ptr, self.f_ptr
            else:
                py, pf = C.c_void_p(), C.c_void_p()
                check(L.ggml_b200_ipc_open(C.create_string_buffer(hyq, 64), C.byref(py)), "ipc_open(y)")
                check(L.ggml_b200_ipc_open(C.create_string_buffer(hfq, 64), C.byref(pf)), "ipc_open(flags)")
                self._opened += [py, pf]
            ys.append(py.value); fs.append(pf.value)
        self.ga = []
        for sl in range(slots):
            ga = Gather()
            ga.world, ga.rank, ga.row_offset, ga.epoch = world, rank, sl * m_total + row_offset, 0
            for q in range(world):
                ga.y_peers[q] = ys[q]; ga.flag_peers[q] = fs[q]
            self.ga.append(ga)
        dist.barrier()

    def mul_mat_gather(self, args: MulMatArgs, slot: int = 0):
        """compute this rank's rows and store them into every peer's gathered y (slot); publishes one exchange epoch"""
        check(lib().ggml_b200_mul_mat_gather(C.byref(args), C.byref(self.ga[slot]), _stream()), "ggml_b200_mul_mat_gather")

    def wait(self):
        """stream-wait until every rank has published as many exchanges as this rank has"""
        check(lib().ggml_b200_gather_wait(self.f_ptr, self.world, 0, _stream()), "ggml_b200_gather_wait")

    def y_full(self, slot: int = 0):
        """zero-copy torch view of this rank's gathered y (slot)"""
        import torch

        class _View:
            pass
        v = _View()
        v.__cuda_array_interface__ = {"shape": (self.m_total,), "typestr": "<f4", "version": 2,
                                      "data": (self.y_ptr.value + slot * self.m_total * 4, False)}
        return torch.as_tensor(v, device="cuda")

    def close(self):
        import torch
        torch.cuda.synchronize()
        for p in self._opened:
            lib().ggml_b200_ipc_close(p)
        lib().ggml_b200_ipc_free(self.y_ptr)
        lib().ggml_b200_ipc_free(self.f_ptr)


# ---------------------------------------------------------------------------------------------------------------
# fused epilogue / small ops used by the backend's graph-level fusion (thin ctypes mirrors, for the tests)
class Epilogue(C.Structure):
    _fields_ = [("bias", C.c_void_p), ("dst_bias", C.c_void_p), ("unary", C.c_int32), ("dst_unary", C.c_void_p), ("residual", C.c_void_p)]


class TensorDesc(C.Structure):
    _fields_ = [("data", C.c_void_p), ("type", C.c_int32), ("ne", C.c_int64 * 4), ("nb", C.c_size_t * 4)]


def tensor_desc(t) -> TensorDesc:
    """descriptor of a contiguous torch tensor in ggml order (ne[0] = last torch dim)"""
    import torch
    d = TensorDesc()
    d.data = t.data_ptr()
    d.type = {torch.float32: F32, torch.float16: F16, torch.int32: 26, torch.int16: 25, torch.bfloat16: 30, torch.int64: 27}[t.dtype]
    shape = list(t.shape)[::-1] + [1] * (4 - t.dim())
    es = t.element_size()
    nb = es
    for i in range(4):
        d.ne[i] = shape[i]
        d.nb[i] = nb
        nb *= shape[i]
    return d


def mul_mat_fused(t, W, X, M, K, bias, gelu: bool, residual=None, out=None, workspace=None):
    """y = W.x ; y2 = y + bias ; y3 = gelu(y2) (or y2 + residual) in one launch (n = 1).  Returns (y, y2, y3 or None).
    out: None (new tensors) or (y, y2, y3) f32 tensors of M elements (y3 None without gelu or residual); workspace: as for mul_mat."""
    import torch
    L = lib()
    L.ggml_b200_mul_mat_fused.argtypes = [C.POINTER(MulMatArgs), C.POINTER(Epilogue), C.c_void_p]
    if out is not None:
        Y, Y2, Y3 = out[0].view(1, 1, 1, M), out[1], out[2]
    else:
        Y = torch.empty((1, 1, 1, M), dtype=torch.float32, device="cuda")
        Y2 = torch.empty(M, dtype=torch.float32, device="cuda")
        Y3 = torch.empty(M, dtype=torch.float32, device="cuda") if (gelu or residual is not None) else None
    a = mul_mat_args(t, W, X, Y, M, 1, K, workspace=workspace)
    ep = Epilogue()
    ep.bias, ep.dst_bias, ep.unary, ep.dst_unary = bias.data_ptr(), Y2.data_ptr(), (2 if residual is not None else 1 if gelu else 0), (Y3.data_ptr() if Y3 is not None else None)
    ep.residual = residual.data_ptr() if residual is not None else None
    check(L.ggml_b200_mul_mat_fused(C.byref(a), C.byref(ep), _stream()), "ggml_b200_mul_mat_fused")
    return Y.view(-1), Y2, Y3


UNARY_SIN, UNARY_COS = 11, 12                  # GGML_B200_UNARY_SIN / _COS (GGML_OP_SIN / GGML_OP_COS): sinf / cosf
UNARY_STEP = 13                                # GGML_B200_UNARY_STEP (GGML_UNARY_OP_STEP): x > 0 ? 1 : 0


def op_unary(uop: int, x):
    import torch
    L = lib()
    L.ggml_b200_op_unary.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    y = torch.empty_like(x)
    check(L.ggml_b200_op_unary(uop, x.data_ptr(), y.data_ptr(), x.numel(), _stream()), "ggml_b200_op_unary")
    return y


def op_norm(x, eps: float, rms: bool = False, out=None):
    """GGML_OP_NORM / RMS_NORM along the last dim of an f32 x (any view with that dim contiguous) -> a new contiguous tensor, or into
    out (a contiguous tensor of x's shape)"""
    import torch
    L = lib()
    L.ggml_b200_op_norm.argtypes = [C.c_int32, C.POINTER(TensorDesc), C.POINTER(TensorDesc), C.c_float, C.c_void_p]
    y = out if out is not None else torch.empty(x.shape, dtype=x.dtype, device=x.device)
    s, d = strided_desc(x), tensor_desc(y)
    check(L.ggml_b200_op_norm(int(rms), C.byref(s), C.byref(d), eps, _stream()), "ggml_b200_op_norm")
    return y


def op_norm_affine(x, gain, bias, eps: float, rms: bool = False):
    import torch
    L = lib()
    L.ggml_b200_op_norm_affine.argtypes = [C.c_int32, C.POINTER(TensorDesc), C.POINTER(TensorDesc), C.c_void_p, C.POINTER(TensorDesc),
                                           C.c_void_p, C.POINTER(TensorDesc), C.c_float, C.c_void_p]
    y1, y2, y3 = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    s, d1, d2, d3 = tensor_desc(x), tensor_desc(y1), tensor_desc(y2), tensor_desc(y3)
    check(L.ggml_b200_op_norm_affine(int(rms), C.byref(s), C.byref(d1), gain.data_ptr(), C.byref(d2), bias.data_ptr(), C.byref(d3), eps, _stream()),
          "ggml_b200_op_norm_affine")
    return y1, y2, y3


def op_scale(x, s: float):
    import torch
    L = lib()
    L.ggml_b200_op_scale.argtypes = [C.c_void_p, C.c_void_p, C.c_float, C.c_int64, C.c_void_p]
    y = torch.empty_like(x)
    check(L.ggml_b200_op_scale(x.data_ptr(), y.data_ptr(), s, x.numel(), _stream()), "ggml_b200_op_scale")
    return y


def op_diag_mask_inf(x, n_past: int):
    """x: [..., ne1, ne0] contiguous f32"""
    import torch
    L = lib()
    L.ggml_b200_op_diag_mask_inf.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_void_p]
    y = torch.empty_like(x)
    check(L.ggml_b200_op_diag_mask_inf(x.data_ptr(), y.data_ptr(), x.shape[-1], x.shape[-2], x.numel(), n_past, _stream()), "ggml_b200_op_diag_mask_inf")
    return y


def op_soft_max(x, scale: float = 1.0, diag_n_past: int = -1, mask=None, max_bias: float = 0.0, inplace: bool = False):
    """row softmax of a contiguous f32 [ne3?, ne2, ne1, ne0] tensor; diag_n_past >= 0: the fused SCALE -> DIAG_MASK_INF -> SOFT_MAX pass.
    mask: a contiguous f16 or f32 [ne01 >= ne1, ne0] added (times the ALiBi slope of head i2 when max_bias > 0) to row i1 of every matrix,
    as ggml_soft_max_ext broadcasts it.  inplace: the result is written into x."""
    import torch
    L = lib()
    L.ggml_b200_op_soft_max_diag.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p] + [C.c_int64] * 4 + [C.c_float, C.c_float, C.c_int32, C.c_void_p]
    sh = [1] * (4 - x.dim()) + list(x.shape)
    y = x if inplace else torch.empty_like(x)
    mp, mt = (None, 0) if mask is None else (mask.data_ptr(), {torch.float32: F32, torch.float16: F16}[mask.dtype])
    check(L.ggml_b200_op_soft_max_diag(x.data_ptr(), mp, mt, y.data_ptr(), sh[3], sh[2], sh[1], sh[0], scale, max_bias, diag_n_past, _stream()),
          "ggml_b200_op_soft_max_diag")
    return y


def op_cpy(src, dst):
    """GGML_OP_CPY: src and dst torch tensors (any views) or TensorDescs (bytes_desc: a view into a quantized cache)"""
    L = lib()
    L.ggml_b200_op_cpy.argtypes = [C.POINTER(TensorDesc), C.POINTER(TensorDesc), C.c_void_p]
    s, d = (t if isinstance(t, TensorDesc) else strided_desc(t) for t in (src, dst))
    check(L.ggml_b200_op_cpy(C.byref(s), C.byref(d), _stream()), "ggml_b200_op_cpy")


def op_cpy2(src_a, dst_a, src_b, dst_b):
    L = lib()
    L.ggml_b200_op_cpy2.argtypes = [C.POINTER(TensorDesc)] * 4 + [C.c_void_p]
    a, b, c, d = tensor_desc(src_a), tensor_desc(dst_a), tensor_desc(src_b), tensor_desc(dst_b)
    check(L.ggml_b200_op_cpy2(C.byref(a), C.byref(b), C.byref(c), C.byref(d), _stream()), "ggml_b200_op_cpy2")


class RopeParams(C.Structure):
    """ggml_b200_rope_params (include/ggml-b200.h)"""
    _fields_ = [("n_dims", C.c_int32), ("mode", C.c_int32), ("sections", C.c_int32 * 4), ("freq_scale", C.c_float), ("ext_factor", C.c_float),
                ("mscale", C.c_float), ("theta_scale", C.c_float), ("corr_dims", C.c_float * 2)]


ROPE_NORM, ROPE_NEOX, ROPE_MROPE, ROPE_VISION = 0, 2, 8, 24


def _libm():
    m = C.CDLL("libm.so.6")
    for fn in ("powf", "logf", "floorf", "ceilf"):
        getattr(m, fn).restype = C.c_float
    m.powf.argtypes = [C.c_float, C.c_float]
    m.logf.argtypes = m.floorf.argtypes = m.ceilf.argtypes = [C.c_float]
    return m


def rope_params(n_dims: int, mode: int = ROPE_NORM, sections=(0, 0, 0, 0), n_ctx_orig: int = 0, freq_base: float = 10000.0, freq_scale: float = 1.0,
                ext_factor: float = 0.0, attn_factor: float = 1.0, beta_fast: float = 32.0, beta_slow: float = 1.0) -> RopeParams:
    """the per-op constants of a ROPE node, derived as the CPU backend derives them: f32 arithmetic and the C library's powf / logf
    (theta_scale = powf(freq_base, -2/n_dims), the YaRN corr dims of ggml_rope_yarn_corr_dims, mscale = attn_factor * (1 + 0.1 logf(1/freq_scale))
    when ext_factor != 0).  theta_scale must be bit-exact: the kernel raises it to the power of the pair index by repeated multiplication."""
    import numpy as np
    f, m = np.float32, _libm()
    p = RopeParams()
    p.n_dims, p.mode = n_dims, mode
    for i in range(4):
        p.sections[i] = int(sections[i])
    p.freq_scale, p.ext_factor = freq_scale, ext_factor
    with np.errstate(divide="ignore", invalid="ignore"):
        p.theta_scale = m.powf(freq_base, float(f(-2.0) / f(n_dims)))

        def corr_dim(n_rot):
            return f(f(n_dims) * f(m.logf(float(f(n_ctx_orig) / (f(n_rot) * f(2) * f(np.pi)))))) / (f(2) * f(m.logf(freq_base)))
        start, end = m.floorf(float(corr_dim(beta_fast))), m.ceilf(float(corr_dim(beta_slow)))
    p.corr_dims[0] = max(0.0, start)
    p.corr_dims[1] = min(float(n_dims - 1), end)
    ms = f(attn_factor)
    if ext_factor != 0.0:
        ms = ms * (f(1) + f(0.1) * f(m.logf(float(f(1) / f(freq_scale)))))
    p.mscale = float(ms)
    return p


def op_rope(x, pos, params: RopeParams, freq_factors=None, inplace: bool = False):
    """GGML_OP_ROPE on a contiguous f32 / f16 torch tensor [ne3, n_pos, n_head, ne0] (ggml order reversed) with i32 positions `pos`
    ([n_pos], or [4 * n_pos] for MROPE / VISION) and optional f32 freq_factors; params from rope_params().  inplace: dst is x."""
    import torch
    L = lib()
    L.ggml_b200_op_rope.argtypes = [C.POINTER(TensorDesc)] * 4 + [C.POINTER(RopeParams), C.c_void_p]
    y = x if inplace else torch.empty_like(x)
    s, p, d = tensor_desc(x), tensor_desc(pos), tensor_desc(y)
    f = C.byref(tensor_desc(freq_factors)) if freq_factors is not None else None
    check(L.ggml_b200_op_rope(C.byref(s), C.byref(p), f, C.byref(d), C.byref(params), _stream()), "ggml_b200_op_rope")
    return y


def op_argsort(x, descending: bool = False):
    """GGML_OP_ARGSORT of a contiguous f32 torch tensor along its last dim (ggml's ne0, <= 1024): int32 indices of the same shape.
    Ties come out in ascending index and NaNs last, so every row is a permutation."""
    import torch
    L = lib()
    L.ggml_b200_op_argsort.argtypes = [C.POINTER(TensorDesc), C.POINTER(TensorDesc), C.c_int32, C.c_void_p]
    y = torch.empty(x.shape, dtype=torch.int32, device=x.device)
    s, d = tensor_desc(x), tensor_desc(y)
    check(L.ggml_b200_op_argsort(C.byref(s), C.byref(d), int(descending), _stream()), "ggml_b200_op_argsort")
    return y


def op_sum_rows(x):
    """GGML_OP_SUM_ROWS of a contiguous f32 torch tensor: the sums over its last dim (accumulated in double), shape [..., 1]"""
    import torch
    L = lib()
    L.ggml_b200_op_sum_rows.argtypes = [C.POINTER(TensorDesc), C.POINTER(TensorDesc), C.c_void_p]
    y = torch.empty(tuple(x.shape[:-1]) + (1,), dtype=torch.float32, device=x.device)
    s, d = tensor_desc(x), tensor_desc(y)
    check(L.ggml_b200_op_sum_rows(C.byref(s), C.byref(d), _stream()), "ggml_b200_op_sum_rows")
    return y


def strided_desc(t) -> TensorDesc:
    """descriptor of a torch tensor with any strides (a view) in ggml order: ne[i] / nb[i] from the torch dim ndim - 1 - i"""
    import torch
    d = TensorDesc()
    d.data = t.data_ptr()
    d.type = {torch.float32: F32, torch.float16: F16, torch.int32: 26, torch.int16: 25, torch.bfloat16: 30, torch.int64: 27}[t.dtype]
    es = t.element_size()
    shape, strides = list(t.shape)[::-1], list(t.stride())[::-1]
    for i in range(4):
        d.ne[i] = shape[i] if i < len(shape) else 1
        d.nb[i] = strides[i] * es if i < len(shape) else (d.nb[i - 1] * d.ne[i - 1] if i else es)
    return d


def bytes_desc(buf, type_: int, ne, nb, offset: int = 0) -> TensorDesc:
    """descriptor of `type_` elements (block-quantized rows too) in the raw bytes of a cuda uint8 tensor, from byte `offset`, with ne[4]
    and nb[4] in ggml order given explicitly: a view into a KV cache, as a graph's ggml_view_4d makes it"""
    d = TensorDesc()
    d.data, d.type = buf.data_ptr() + offset, type_
    for i in range(4):
        d.ne[i], d.nb[i] = ne[i], nb[i]
    return d


def op_flash_attn_ext(q, k, v, mask, scale: float, max_bias: float = 0.0, softcap: float = 0.0):
    """GGML_OP_FLASH_ATTN_EXT: q f32 [ne3, n_head, n_q, D] (torch order of ggml's [D, n_q, n_head, ne3]; any view with the last dim
    contiguous, e.g. a permuted one); k and v [nk3, n_head_kv, n_kv, D], torch tensors or TensorDescs (bytes_desc: block rows of a cache
    view); mask None or f16 [>= n_q, n_kv'] with n_kv' >= n_kv (row i for query i).  Returns a new f32 tensor [ne3, n_q, n_head, D]
    (ggml's [D, n_head, n_q, ne3])."""
    import torch
    ne3, n_head, n_q, D = q.shape
    y = torch.empty((ne3, n_q, n_head, D), dtype=torch.float32, device=q.device)
    descs = [strided_desc(q)] + [t if isinstance(t, TensorDesc) else strided_desc(t) for t in (k, v)]
    L = lib()
    L.ggml_b200_op_flash_attn_ext.argtypes = [C.POINTER(TensorDesc)] * 5 + [C.c_float] * 3 + [C.c_void_p]
    m = C.byref(strided_desc(mask)) if mask is not None else None
    check(L.ggml_b200_op_flash_attn_ext(*(C.byref(d) for d in descs), m, C.byref(tensor_desc(y)), scale, max_bias, softcap, _stream()),
          "ggml_b200_op_flash_attn_ext")
    return y


def op_mul_mat_f(a, b, out=None):
    """the float GGML_OP_MUL_MAT (KQ and KQV of non-flash attention): a f32 or f16 [a3, a2, M, K], b f32 (f16 with an f16 a) [b3, b2, N, K],
    both any views (a transposed V: nb0 != the element size); a's batch dims broadcast over b's.  out: None (a new contiguous tensor) or an
    f32 tensor [b3, b2, N, M] of any strides.  out[.., n, m] = sum_k a[.., m, k] b[.., n, k], b rounded to f16 first when a is f16 and b f32."""
    import torch
    y = out if out is not None else torch.empty(tuple(b.shape[:-1]) + (a.shape[-2],), dtype=torch.float32, device=a.device)
    _launch("ggml_b200_op_mul_mat_f", strided_desc(a), strided_desc(b), strided_desc(y))
    return y


def op_concat(a, b, dim: int):
    """GGML_OP_CONCAT of two f32 (or two i32) torch tensors of equal rank <= 4 along ggml's dim (0 = the last torch dim): a, then b.
    a must be contiguous along its last dim; b may be any view (a transposed one, as in the Mamba layer).  A new contiguous tensor."""
    import torch
    L = lib()
    L.ggml_b200_op_concat.argtypes = [C.POINTER(TensorDesc)] * 3 + [C.c_int32, C.c_void_p]
    shape = list(a.shape)
    if 0 <= dim < a.dim():
        shape[a.dim() - 1 - dim] += b.shape[a.dim() - 1 - dim]
    y = torch.empty(shape, dtype=a.dtype, device=a.device)
    s0, s1, d = strided_desc(a), strided_desc(b), tensor_desc(y)
    check(L.ggml_b200_op_concat(C.byref(s0), C.byref(s1), C.byref(d), int(dim), _stream()), "ggml_b200_op_concat")
    return y


def op_ssm_conv(sx, c):
    """GGML_OP_SSM_CONV: sx f32 [n_s, d_inner, d_conv - 1 + n_t] (rows packed), c f32 [d_inner, d_conv] -> f32 [n_s, n_t, d_inner],
    out[s, t, i] = sum_k sx[s, i, t + k] * c[i, k], bit-identical to ggml-cpu"""
    import torch
    L = lib()
    L.ggml_b200_op_ssm_conv.argtypes = [C.POINTER(TensorDesc)] * 3 + [C.c_void_p]
    n_s, d_inner, ncs = sx.shape
    y = torch.empty((n_s, ncs - c.shape[-1] + 1, d_inner), dtype=torch.float32, device=sx.device)
    x, w, d = strided_desc(sx), strided_desc(c), tensor_desc(y)
    check(L.ggml_b200_op_ssm_conv(C.byref(x), C.byref(w), C.byref(d), _stream()), "ggml_b200_op_ssm_conv")
    return y


def op_ssm_scan(s, x, dt, A, B, C_):
    """GGML_OP_SSM_SCAN (Mamba-1): s f32 [n_s, d_inner, d_state], x and dt f32 [n_s, n_t, d_inner], A f32 [d_inner, d_state] (all four
    contiguous), B and C f32 [n_s, n_t, d_state] (last dim contiguous, any other strides).  Returns (y [n_s, n_t, d_inner], s_new
    [n_s, d_inner, d_state]): views of the one flat result in ggml's layout (y, then the final states)."""
    import torch
    L = lib()
    L.ggml_b200_op_ssm_scan.argtypes = [C.POINTER(TensorDesc)] * 7 + [C.c_void_p]
    out = torch.empty(x.numel() + s.numel(), dtype=torch.float32, device=x.device)
    t = [strided_desc(v) for v in (s, x, dt, A, B, C_)]
    d = tensor_desc(out)
    check(L.ggml_b200_op_ssm_scan(*[C.byref(v) for v in t], C.byref(d), _stream()), "ggml_b200_op_ssm_scan")
    return out[: x.numel()].view(x.shape), out[x.numel():].view(s.shape)


def _wkv(fn, name, k, s, srcs, extra):
    """the flat ggml result of RWKV_WKV6 / GATED_LINEAR_ATTN as (y [T, H, S], s_new [n_seqs, H, S, S]) views; s is read as [n_seqs, S S H]"""
    import torch
    T, H, S = k.shape
    n_seqs = s.shape[0]
    out = torch.empty((T + S * n_seqs, H * S), dtype=torch.float32, device=k.device)
    t = [strided_desc(v) for v in srcs] + [strided_desc(s.reshape(n_seqs, -1))]
    check(fn(*[C.byref(v) for v in t], C.byref(tensor_desc(out)), *extra, _stream()), name)
    return out[:T].view(T, H, S), out[T:].view(n_seqs, H, S, S)


def op_rwkv_wkv6(k, v, r, tf, td, s):
    """GGML_OP_RWKV_WKV6: k, v, r, td f32 [T, H, S], tf f32 [H, S], s f32 [n_seqs, H, S, S] (state[i][j] at [q, h, i, j]), all contiguous;
    sequence q owns tokens [q T / n_seqs, (q + 1) T / n_seqs).  Returns (y [T, H, S], s_new [n_seqs, H, S, S]): views of the one flat
    result in ggml's layout (y, then the final states)."""
    L = lib()
    L.ggml_b200_op_rwkv_wkv6.argtypes = [C.POINTER(TensorDesc)] * 7 + [C.c_void_p]
    return _wkv(L.ggml_b200_op_rwkv_wkv6, "ggml_b200_op_rwkv_wkv6", k, s, (k, v, r, tf, td), ())


def op_gated_linear_attn(k, v, q, g, s, scale: float):
    """GGML_OP_GATED_LINEAR_ATTN: k, v, q, g f32 [T, H, S], s f32 [n_seqs, H, S, S], all contiguous; as op_rwkv_wkv6 with the gate g in
    place of the decay and q * scale in place of r (no bonus term).  Returns (y [T, H, S], s_new [n_seqs, H, S, S])."""
    L = lib()
    L.ggml_b200_op_gated_linear_attn.argtypes = [C.POINTER(TensorDesc)] * 6 + [C.c_float, C.c_void_p]
    return _wkv(L.ggml_b200_op_gated_linear_attn, "ggml_b200_op_gated_linear_attn", k, s, (k, v, q, g), (float(scale),))


class Im2colParams(C.Structure):
    """ggml_b200_im2col_params (include/ggml-b200.h)"""
    _fields_ = [("s0", C.c_int32), ("s1", C.c_int32), ("p0", C.c_int32), ("p1", C.c_int32), ("d0", C.c_int32), ("d1", C.c_int32), ("is_2D", C.c_int32)]


def conv_out_size(ins: int, ks: int, s: int, p: int, d: int) -> int:
    """the output extent of a convolution along one axis (ggml_calc_conv_output_size)"""
    return (ins + 2 * p - d * (ks - 1) - 1) // s + 1


def op_im2col(kernel, x, s0: int, p0: int, d0: int, s1: int = 1, p1: int = 0, d1: int = 1, is_2d: bool = False, dtype=None):
    """GGML_OP_IM2COL (the first node of ggml_conv_1d / ggml_conv_2d): kernel [OC, IC, KW] (2-D: [OC, IC, KH, KW]; only its shape is read, and
    its dtype, which must be float16 for a float16 result), x f32 [N, IC, IW] (2-D: [N, IC, IH, IW]; last dim contiguous, any other strides)
    -> a new contiguous tensor [N, OW, IC KW] (2-D: [N, OH, OW, IC KH KW]) of `dtype` (default float16, as ggml_conv_1d builds it),
    bit-identical to ggml-cpu"""
    import torch
    L = lib()
    L.ggml_b200_op_im2col.argtypes = [C.POINTER(TensorDesc)] * 3 + [C.POINTER(Im2colParams), C.c_void_p]
    dtype = torch.float16 if dtype is None else dtype
    kw, ic = kernel.shape[-1], x.shape[1]
    ow = conv_out_size(x.shape[-1], kw, s0, p0, d0)
    if is_2d:
        kh = kernel.shape[-2]
        shape = (x.shape[0], conv_out_size(x.shape[-2], kh, s1, p1, d1), ow, ic * kh * kw)
    else:
        shape = (x.shape[0], ow, ic * kw)
    y = torch.empty(shape, dtype=dtype, device=x.device)
    p = Im2colParams(s0, s1, p0, p1, d0, d1, 1 if is_2d else 0)
    k, s, d = strided_desc(kernel), strided_desc(x), tensor_desc(y)
    check(L.ggml_b200_op_im2col(C.byref(k), C.byref(s), C.byref(d), C.byref(p), _stream()), "ggml_b200_op_im2col")
    return y


def mul_mat_f16_f16_workspace_size(M: int, N: int, K: int) -> int:
    """bytes the tensor-core f16 x f16 GEMM needs for [M, K] x [N, K]; 0 when the shape is not eligible for it"""
    L = lib()
    L.ggml_b200_mul_mat_f16_f16_workspace_size.restype = C.c_size_t
    L.ggml_b200_mul_mat_f16_f16_workspace_size.argtypes = [C.c_int64] * 3
    return int(L.ggml_b200_mul_mat_f16_f16_workspace_size(M, N, K))


def mul_mat_f16_f16(w, x, flags: int = 0, out=None):
    """f16 w [M, K] x f16 x [N, K] (rows contiguous, any row stride that is a multiple of 16 bytes) -> f32 [N, M] on the tensor cores
    (ggml_b200_mul_mat_f16_f16); raises when the shape is not eligible (N >= 9, K % 64 == 0)"""
    import torch
    L = lib()
    L.ggml_b200_mul_mat_f16_f16.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                            C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    M, K = w.shape
    N = x.shape[0]
    need = mul_mat_f16_f16_workspace_size(M, N, K)
    if need == 0:
        raise B200Error(f"mul_mat_f16_f16: ({M}, {N}, {K}) is not eligible for the tensor-core path")
    y = out if out is not None else torch.empty((N, M), dtype=torch.float32, device=w.device)
    ws = _ws.get(need)
    check(L.ggml_b200_mul_mat_f16_f16(w.data_ptr(), w.stride(0) * 2, x.data_ptr(), x.stride(0) * 2, y.data_ptr(), M, N, K, ws.data_ptr(), ws.numel(),
                                      flags, _stream()), "ggml_b200_mul_mat_f16_f16")
    return y


class PoolParams(C.Structure):
    """ggml_b200_pool_params (include/ggml-b200.h)"""
    _fields_ = [("op", C.c_int32), ("k0", C.c_int32), ("k1", C.c_int32), ("s0", C.c_int32), ("s1", C.c_int32), ("p0", C.c_int32), ("p1", C.c_int32)]


POOL_MAX, POOL_AVG = 0, 1


def pool_out_size(ins: int, ks: int, s: int, p: float) -> int:
    """the output extent of a pool along one axis as ggml_calc_pool_output_size computes it: in float, from the float padding"""
    import numpy as np
    f = np.float32
    return int((f(ins) + f(2) * f(p) - f(ks)) / f(s) + f(1))


def op_pool_2d(x, op: int, k0: int, k1: int, s0: int, s1: int, p0: float = 0.0, p1: float = 0.0):
    """GGML_OP_POOL_2D (ggml_pool_2d): x f32 [N, C, IH, IW] (last dim contiguous, any other strides), op POOL_MAX or POOL_AVG, window k0 x k1
    (width x height), stride s0 / s1, paddings p0 / p1 as ggml_pool_2d takes them (float: they size the output, and the kernel uses them
    truncated, as ggml-cpu does) -> a new contiguous f32 tensor [N, C, OH, OW], bit-identical to ggml-cpu"""
    import torch
    L = lib()
    L.ggml_b200_op_pool_2d.argtypes = [C.POINTER(TensorDesc)] * 2 + [C.POINTER(PoolParams), C.c_void_p]
    oh, ow = pool_out_size(x.shape[-2], k1, s1, p1), pool_out_size(x.shape[-1], k0, s0, p0)
    y = torch.empty(tuple(x.shape[:-2]) + (oh, ow), dtype=torch.float32, device=x.device)
    p = PoolParams(int(op), k0, k1, s0, s1, int(p0), int(p1))
    s, d = strided_desc(x), tensor_desc(y)
    check(L.ggml_b200_op_pool_2d(C.byref(s), C.byref(d), C.byref(p), _stream()), "ggml_b200_op_pool_2d")
    return y


def op_upscale(x, shape):
    """GGML_OP_UPSCALE (nearest; ggml_upscale_ext): x f32 of rank <= 4, any strides -> a new contiguous f32 tensor of `shape` (same rank,
    every extent >= x's; torch order), element i = x[i * x.shape / shape] per dim with ggml-cpu's float factors, bit-identical.
    ggml_upscale(x, f) is shape = x.shape with the last two dims times f."""
    import torch
    L = lib()
    L.ggml_b200_op_upscale.argtypes = [C.POINTER(TensorDesc)] * 2 + [C.c_void_p]
    y = torch.empty(tuple(shape), dtype=torch.float32, device=x.device)
    s, d = strided_desc(x), tensor_desc(y)
    check(L.ggml_b200_op_upscale(C.byref(s), C.byref(d), _stream()), "ggml_b200_op_upscale")
    return y


def op_leaky_relu(x, slope: float, inplace: bool = False):
    """GGML_OP_LEAKY_RELU of an f32 torch tensor (last dim contiguous, any other strides): ((x > 0) ? x : 0) + slope ((x < 0) ? x : 0),
    bit-identical to ggml-cpu (NaN and -0 give +0).  inplace: the result is written into x."""
    import torch
    L = lib()
    L.ggml_b200_op_leaky_relu.argtypes = [C.POINTER(TensorDesc)] * 2 + [C.c_float, C.c_void_p]
    y = x if inplace else torch.empty(x.shape, dtype=torch.float32, device=x.device)
    s, d = strided_desc(x), strided_desc(y)
    check(L.ggml_b200_op_leaky_relu(C.byref(s), C.byref(d), float(slope), _stream()), "ggml_b200_op_leaky_relu")
    return y


def op_repeat(x, shape):
    """GGML_OP_REPEAT: x (float32, int32, float16, bfloat16 or int16; last dim contiguous, any other strides) tiled into a new contiguous
    tensor of `shape` (torch order, each extent a whole multiple of x's), copied as raw words: every bit pattern is kept"""
    import torch
    L = lib()
    L.ggml_b200_op_repeat.argtypes = [C.POINTER(TensorDesc)] * 2 + [C.c_void_p]
    y = torch.empty(tuple(shape), dtype=x.dtype, device=x.device)
    s, d = strided_desc(x), strided_desc(y)
    check(L.ggml_b200_op_repeat(C.byref(s), C.byref(d), _stream()), "ggml_b200_op_repeat")
    return y


def op_win_part(x, w: int):
    """GGML_OP_WIN_PART (ggml_win_part): x f32 [H0, W0, C] (packed; torch order of ggml's [C, W0, H0]) -> a new f32 tensor
    [npx npy, w, w, C], window py npx + px holding pixels (px w + i1, py w + i2), zeros past the image; raw words, bit-identical to ggml-cpu"""
    import torch
    L = lib()
    L.ggml_b200_op_win_part.argtypes = [C.POINTER(TensorDesc)] * 2 + [C.c_int32] * 3 + [C.c_void_p]
    h0, w0, c = x.shape[-3:]
    npx, npy = -(-w0 // w), -(-h0 // w)
    y = torch.empty((npx * npy, w, w, c), dtype=torch.float32, device=x.device)
    s, d = strided_desc(x), tensor_desc(y)
    check(L.ggml_b200_op_win_part(C.byref(s), C.byref(d), npx, npy, w, _stream()), "ggml_b200_op_win_part")
    return y


def op_win_unpart(x, w0: int, h0: int, w: int):
    """GGML_OP_WIN_UNPART (ggml_win_unpart): x f32 [np, w, w, C] (packed, np >= ceil(w0 / w) ceil(h0 / w)) -> a new f32 tensor [h0, w0, C],
    the inverse of op_win_part without its padding; raw words, bit-identical to ggml-cpu"""
    import torch
    L = lib()
    L.ggml_b200_op_win_unpart.argtypes = [C.POINTER(TensorDesc)] * 2 + [C.c_int32, C.c_void_p]
    y = torch.empty((h0, w0, x.shape[-1]), dtype=torch.float32, device=x.device)
    s, d = strided_desc(x), tensor_desc(y)
    check(L.ggml_b200_op_win_unpart(C.byref(s), C.byref(d), w, _stream()), "ggml_b200_op_win_unpart")
    return y


def op_get_rel_pos(x):
    """GGML_OP_GET_REL_POS (ggml_get_rel_pos): x f16 [2w - 1, C] (packed) -> a new f16 tensor [w, w, C], y[i2, i1] = x[(w - 1 - i1) + i2];
    raw 2-byte words, bit-identical to ggml-cpu"""
    import torch
    L = lib()
    L.ggml_b200_op_get_rel_pos.argtypes = [C.POINTER(TensorDesc)] * 2 + [C.c_void_p]
    w = (x.shape[-2] + 1) // 2
    y = torch.empty((w, w, x.shape[-1]), dtype=x.dtype, device=x.device)
    s, d = strided_desc(x), tensor_desc(y)
    check(L.ggml_b200_op_get_rel_pos(C.byref(s), C.byref(d), _stream()), "ggml_b200_op_get_rel_pos")
    return y


def op_add_rel_pos(a, pw, ph, inplace: bool = False):
    """GGML_OP_ADD_REL_POS (ggml_add_rel_pos[_inplace]): a f32 [P, A B, L L], pw and ph f32 [P, B, A, L] (all packed) ->
    a[p, q, kh L + kw] + ph[p, q, kh] + pw[p, q, kw] with ggml-cpu's order of the two adds (ph first when kh <= kw): bit-identical.
    inplace: the result is written into a."""
    import torch
    L = lib()
    L.ggml_b200_op_add_rel_pos.argtypes = [C.POINTER(TensorDesc)] * 4 + [C.c_void_p]
    y = a if inplace else torch.empty(a.shape, dtype=torch.float32, device=a.device)
    s, w, h, d = strided_desc(a), strided_desc(pw), strided_desc(ph), strided_desc(y)
    check(L.ggml_b200_op_add_rel_pos(C.byref(s), C.byref(w), C.byref(h), C.byref(d), _stream()), "ggml_b200_op_add_rel_pos")
    return y


def op_conv_transpose_2d(kernel, x, stride: int):
    """GGML_OP_CONV_TRANSPOSE_2D (ggml_conv_transpose_2d_p0): kernel f16 [Cin, Cout, Kh, Kw] (packed Kh x Kw planes), x f32 [Cin, H, W] or
    [1, Cin, H, W] (last dim contiguous) -> a new f32 tensor [(1,) Cout, (H-1) s + Kh, (W-1) s + Kw], padding 0.  x is rounded to fp16 as
    ggml-cpu rounds it; each tap's dot over Cin is summed in f32 and the taps are added in ggml-cpu's order."""
    import torch
    L = lib()
    L.ggml_b200_op_conv_transpose_2d.argtypes = [C.POINTER(TensorDesc)] * 3 + [C.c_int32, C.c_void_p]
    cout, kh, kw = kernel.shape[1:]
    h, w = x.shape[-2:]
    y = torch.empty(tuple(x.shape[:-3]) + (cout, (h - 1) * stride + kh, (w - 1) * stride + kw), dtype=torch.float32, device=x.device)
    k, s, d = strided_desc(kernel), strided_desc(x), tensor_desc(y)
    check(L.ggml_b200_op_conv_transpose_2d(C.byref(k), C.byref(s), C.byref(d), stride, _stream()), "ggml_b200_op_conv_transpose_2d")
    return y


def op_get_rows(src, ids, out):
    """GGML_OP_GET_ROWS: out[i12, i11, i10, :] = row ids[i12, i11, i10] of src's matrix (i11, i12), decoded to f32.  src a torch tensor
    (any view with packed rows) or a TensorDesc (bytes_desc: block-quantized rows), ggml [ne0, rows, ne11, ne12]; ids i32 [ne12, ne11, n],
    any view; out f32 [ne12, ne11, n, ne0], any view with packed rows (a padded row stride)"""
    _launch("ggml_b200_op_get_rows", src if isinstance(src, TensorDesc) else strided_desc(src), strided_desc(ids), strided_desc(out))
    return out


def op_bin_bcast(op: int, a, b, out=None):
    """GGML_OP_ADD / MUL / SUB / DIV (op 0 / 1 / 2 / 3) of f32 a and b, b's dims dividing a's (ggml's whole-repeat broadcast); a, b and out
    any views (out = a: in place).  out None: a new contiguous tensor"""
    import torch
    y = out if out is not None else torch.empty(a.shape, dtype=torch.float32, device=a.device)
    L = lib()
    L.ggml_b200_op_bin_bcast.argtypes = [C.c_int32] + [C.POINTER(TensorDesc)] * 3 + [C.c_void_p]
    s0, s1, d = strided_desc(a), strided_desc(b), strided_desc(y)
    check(L.ggml_b200_op_bin_bcast(op, C.byref(s0), C.byref(s1), C.byref(d), _stream()), "ggml_b200_op_bin_bcast")
    return y


def _launch(name: str, *descs):
    L = lib()
    fn = getattr(L, name)
    fn.argtypes = [C.POINTER(TensorDesc)] * len(descs) + [C.c_void_p]
    check(fn(*(C.byref(d) for d in descs), _stream()), name)


def op_out_prod(a, b):
    """GGML_OP_OUT_PROD (ggml_out_prod): a f32 torch [(b3,) (b2,) K, M] with its last dim contiguous, b f32 torch [(B3,) (B2,) K, N] with any
    strides (b.t() of a contiguous [N, K] is the gradient's form) -> a new f32 tensor [(B3,) (B2,) N, M], out[.., n, m] = sum_k a[.., k, m]
    b[.., k, n]: one fused multiply-add per term in ascending k; a's batch dims broadcast over b's as in MUL_MAT"""
    import torch
    y = torch.empty(tuple(b.shape[:-2]) + (b.shape[-1], a.shape[-1]), dtype=torch.float32, device=a.device)
    _launch("ggml_b200_op_out_prod", strided_desc(a), strided_desc(b), tensor_desc(y))
    return y


def op_cross_entropy_loss(logits, labels):
    """GGML_OP_CROSS_ENTROPY_LOSS: logits and labels f32 of one shape (rows = the last dim, contiguous) -> a new f32 tensor [1]:
    -1/nr sum of labels * log_softmax(logits), reduced in one fixed order"""
    import torch
    y = torch.empty((1,), dtype=torch.float32, device=logits.device)
    _launch("ggml_b200_op_cross_entropy_loss", strided_desc(logits), strided_desc(labels), tensor_desc(y))
    return y


def op_cross_entropy_loss_back(grad, logits, labels):
    """GGML_OP_CROSS_ENTROPY_LOSS_BACK: grad f32 [1] (read on the device), logits and labels f32 of one shape, contiguous -> a new tensor
    (softmax(logits) - labels) * grad / nr, row by row"""
    import torch
    y = torch.empty_like(logits)
    _launch("ggml_b200_op_cross_entropy_loss_back", tensor_desc(grad), tensor_desc(logits), tensor_desc(labels), tensor_desc(y))
    return y


def op_opt_step_adamw(w, g, m, v, params):
    """GGML_OP_OPT_STEP_ADAMW, in place on w, m and v (f32, contiguous, one shape) with the gradient g; params f32 [7] on the device =
    alpha, beta1, beta2, eps, wd, beta1h, beta2h, read by the kernel; bit-identical to ggml-cpu.  Returns w."""
    _launch("ggml_b200_op_opt_step_adamw", tensor_desc(w), tensor_desc(g), tensor_desc(m), tensor_desc(v), tensor_desc(params))
    return w


def op_argmax(x):
    """GGML_OP_ARGMAX: x f32 [rows, n] (last dim contiguous) -> a new i32 tensor [rows], ggml-cpu's rule: the last index of the maximum,
    a NaN restarting the search, a trailing run of NaNs ignored, 0 for a row of NaNs"""
    import torch
    y = torch.empty((x.shape[0],), dtype=torch.int32, device=x.device)
    _launch("ggml_b200_op_argmax", strided_desc(x), tensor_desc(y))
    return y


def op_count_equal(a, b):
    """GGML_OP_COUNT_EQUAL: a and b i32 of one shape, at most 2-D (any strides) -> a new i64 tensor [1], the number of equal pairs"""
    import torch
    y = torch.empty((1,), dtype=torch.int64, device=a.device)
    _launch("ggml_b200_op_count_equal", strided_desc(a), strided_desc(b), tensor_desc(y))
    return y


def op_sum(x):
    """GGML_OP_SUM: x f32 (last dim contiguous) -> a new f32 tensor [1], the sum in double rounded once"""
    import torch
    y = torch.empty((1,), dtype=torch.float32, device=x.device)
    _launch("ggml_b200_op_sum", strided_desc(x), tensor_desc(y))
    return y


def op_repeat_back(x, shape):
    """GGML_OP_REPEAT_BACK: x f32 (last dim contiguous, any other strides) -> a new f32 tensor of `shape` (torch order), each of whose
    extents divides x's: the sum over the repeats, in ggml-cpu's order (bit-identical)"""
    import torch
    y = torch.empty(tuple(shape), dtype=torch.float32, device=x.device)
    _launch("ggml_b200_op_repeat_back", strided_desc(x), tensor_desc(y))
    return y
