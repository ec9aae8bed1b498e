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


def mul_mat_args(t, W, X, Y, M, N, K, batch=(1, 1, 1, 1), flags=MM_AUTO, nb=None) -> MulMatArgs:
    """W: cuda uint8 tensor of packed blocks; X: cuda float32; Y: cuda float32 [ne13, ne12, N, M]."""
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
    need = int(lib().ggml_b200_mul_mat_workspace_size(C.byref(a)))
    ws = _ws.get(need)
    a.workspace, a.workspace_size = ws.data_ptr(), ws.numel()
    return a


def mul_mat(t, W, X, M, N, K, batch=(1, 1, 1, 1), flags=MM_AUTO, out=None, nb=None):
    """GGML_OP_MUL_MAT on the current CUDA stream.  Returns Y[ne13, ne12, N, M] (float32, cuda)."""
    import torch
    ne02, ne03, ne12, ne13 = batch
    Y = out if out is not None else torch.empty((ne13, ne12, N, M), dtype=torch.float32, device="cuda")
    a = mul_mat_args(t, W, X, Y, M, N, K, batch, flags, nb)
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


def mul_mat_id(t, W, X, ids, M, K, n_expert, n_used, nb1cols, n_tok):
    """GGML_OP_MUL_MAT_ID.  W: packed [n_expert, M, row]; X: f32 [n_tok, nb1cols, K]; ids: int32 [n_tok, >= n_used]."""
    import torch
    Y = torch.empty((n_tok, n_used, M), dtype=torch.float32, device="cuda")
    rb = row_size(t, K)
    a = MulMatIdArgs()
    a.type, a.flags, a.K, a.M = t, 0, K, M
    a.n_expert, a.n_used, a.nb1cols, a.n_tok = n_expert, n_used, nb1cols, n_tok
    a.nb01, a.nb02, a.nb11, a.nb12 = rb, rb * M, K * 4, K * 4 * nb1cols
    a.ids_nb1 = ids.stride(0) * 4
    a.src0, a.src1, a.ids, a.dst = W.data_ptr(), X.data_ptr(), ids.data_ptr(), Y.data_ptr()
    need = int(lib().ggml_b200_mul_mat_id_workspace_size(C.byref(a)))
    ws = _ws.get(need)
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
    d.type = {torch.float32: F32, torch.float16: F16, torch.int32: 26}[t.dtype]
    shape = list(t.shape)[::-1] + [1] * (4 - t.dim())
    es = t.element_size()
    nb = es
    for i in range(4):
        d.ne[i] = shape[i]
        d.nb[i] = nb
        nb *= shape[i]
    return d


def mul_mat_fused(t, W, X, M, K, bias, gelu: bool, residual=None):
    """y = W.x ; y2 = y + bias ; y3 = gelu(y2) (or y2 + residual) in one launch (n = 1).  Returns (y, y2, y3 or None)."""
    import torch
    L = lib()
    L.ggml_b200_mul_mat_fused.argtypes = [C.POINTER(MulMatArgs), C.POINTER(Epilogue), C.c_void_p]
    Y = torch.empty((1, 1, 1, M), dtype=torch.float32, device="cuda")
    Y2 = torch.empty(M, dtype=torch.float32, device="cuda")
    Y3 = torch.empty(M, dtype=torch.float32, device="cuda") if (gelu or residual is not None) else None
    a = mul_mat_args(t, W, X, Y, M, 1, K)
    ep = Epilogue()
    ep.bias, ep.dst_bias, ep.unary, ep.dst_unary = bias.data_ptr(), Y2.data_ptr(), (2 if residual is not None else 1 if gelu else 0), (Y3.data_ptr() if Y3 is not None else None)
    ep.residual = residual.data_ptr() if residual is not None else None
    check(L.ggml_b200_mul_mat_fused(C.byref(a), C.byref(ep), _stream()), "ggml_b200_mul_mat_fused")
    return Y.view(-1), Y2, Y3


def op_unary(uop: int, x):
    import torch
    L = lib()
    L.ggml_b200_op_unary.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    y = torch.empty_like(x)
    check(L.ggml_b200_op_unary(uop, x.data_ptr(), y.data_ptr(), x.numel(), _stream()), "ggml_b200_op_unary")
    return y


def op_norm(x, eps: float, rms: bool = False):
    import torch
    L = lib()
    L.ggml_b200_op_norm.argtypes = [C.c_int32, C.POINTER(TensorDesc), C.POINTER(TensorDesc), C.c_float, C.c_void_p]
    y = torch.empty_like(x)
    s, d = tensor_desc(x), tensor_desc(y)
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


def op_soft_max(x, scale: float = 1.0, diag_n_past: int = -1):
    """row softmax of a contiguous f32 [ne3?, ne2, ne1, ne0] tensor; diag_n_past >= 0: the fused SCALE -> DIAG_MASK_INF -> SOFT_MAX pass"""
    import torch
    L = lib()
    L.ggml_b200_op_soft_max_diag.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p] + [C.c_int64] * 4 + [C.c_float, C.c_float, C.c_int32, C.c_void_p]
    sh = [1] * (4 - x.dim()) + list(x.shape)
    y = torch.empty_like(x)
    check(L.ggml_b200_op_soft_max_diag(x.data_ptr(), None, 0, y.data_ptr(), sh[3], sh[2], sh[1], sh[0], scale, 0.0, diag_n_past, _stream()), "ggml_b200_op_soft_max_diag")
    return y


def op_cpy(src, dst):
    L = lib()
    L.ggml_b200_op_cpy.argtypes = [C.POINTER(TensorDesc), C.POINTER(TensorDesc), C.c_void_p]
    s, d = tensor_desc(src), tensor_desc(dst)
    check(L.ggml_b200_op_cpy(C.byref(s), C.byref(d), _stream()), "ggml_b200_op_cpy")


def op_cpy2(src_a, dst_a, src_b, dst_b):
    L = lib()
    L.ggml_b200_op_cpy2.argtypes = [C.POINTER(TensorDesc)] * 4 + [C.c_void_p]
    a, b, c, d = tensor_desc(src_a), tensor_desc(dst_a), tensor_desc(src_b), tensor_desc(dst_b)
    check(L.ggml_b200_op_cpy2(C.byref(a), C.byref(b), C.byref(c), C.byref(d), _stream()), "ggml_b200_op_cpy2")
