"""TEST INFRASTRUCTURE ONLY: GGML_OP_IM2COL and f16 x f16 GGML_OP_MUL_MAT cases and the reference's ops through
oracle/_ref/libggml_conv_probe.so (oracle/conv_probe.cpp).

`Im2colCase` describes one IM2COL node (kernel and input extents, the input's view, stride / padding / dilation, 1-D or 2-D, dst type) and
makes its input from a seed; `im2col_grid()` is the set the CPU (host-compiled b200_conv.cuh) and GPU (device kernel) parity tests run.
`im2col(dev, case)`, `mul_mat_f16(dev, ...)` and `conv_1d(dev, ...)` evaluate on a named ggml device ("CPU": ggml-cpu; "B2000": the
plug-in, once loaded with oracle.Ref().load_backend).  `Im2colCase.view_of_input()` gives the input's parent array with the ne / nb through which
the node reads it, exactly as conv_probe.cpp's input() builds it, so the host emulation reads the same bytes."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from .probe import probe_lib, ptrs, result
from .ssm import View, _nb

F32, F16 = 0, 1


def input_parent_ne(ne, view):
    """the parent shape conv_probe.cpp's input() allocates for an input of shape ne through `view`"""
    ne0, ne1, ne2, ne3 = ne
    pad = 1 if view else 0
    return (ne0 + (5 if view == 2 else 0), ne1 + 3 * pad, ne2 + 2 * pad, ne3)


def conv_out(ins, ks, s, p, d):
    """ggml_calc_conv_output_size"""
    return (ins + 2 * p - d * (ks - 1) - 1) // s + 1


@dataclass
class Im2colCase:
    ne_kernel: tuple            # 1-D: [KW, IC, OC, 1]; 2-D: [KW, KH, IC, OC]
    ne_input: tuple             # 1-D: [IW, IC, N, 1];  2-D: [IW, IH, IC, N]
    s0: int = 1
    s1: int = 1
    p0: int = 0
    p1: int = 0
    d0: int = 1
    d1: int = 1
    is_2d: bool = False
    dst_type: int = F32
    kernel_type: int = F16
    view: int = 0
    seed: int = 0

    @property
    def params(self):
        return np.array([self.s0, self.s1, self.p0, self.p1, self.d0, self.d1, 1 if self.is_2d else 0], dtype=np.int32)

    @property
    def ne_dst(self):
        kw, kh = self.ne_kernel[0], (self.ne_kernel[1] if self.is_2d else 1)
        ic = self.ne_input[2] if self.is_2d else self.ne_input[1]
        ow = conv_out(self.ne_input[0], kw, self.s0, self.p0, self.d0)
        if self.is_2d:
            return (ic * kh * kw, ow, conv_out(self.ne_input[1], kh, self.s1, self.p1, self.d1), self.ne_input[3])
        return (ic * kw, ow, self.ne_input[2], 1)

    def view_of_input(self) -> View:
        """the input as the node reads it: parent array (values from the seed) and ne / nb"""
        rng = np.random.default_rng(11000 + self.seed)
        pne = input_parent_ne(self.ne_input, self.view)
        x = rng.standard_normal(pne[::-1]).astype(np.float32) * np.float32(4.0)
        x.reshape(-1)[3::29] = -0.0                              # signed zeros and values that round to fp16 ties / subnormals / overflow
        x.reshape(-1)[7::31] = np.float32(65520.0)
        x.reshape(-1)[11::37] = np.float32(1.0 + 2.0 ** -11)
        x.reshape(-1)[13::41] = np.float32(3e-6)
        return View(x, tuple(self.ne_input), _nb(pne, 4))

    def __str__(self):
        return (f"im2col {'2d' if self.is_2d else '1d'} k={self.ne_kernel} x={self.ne_input}/v{self.view} s=({self.s0},{self.s1}) "
                f"p=({self.p0},{self.p1}) d=({self.d0},{self.d1}) dst={'f16' if self.dst_type else 'f32'}")


def im2col_grid() -> list:
    """1-D and 2-D, both dst types, strides 1 / 2 / 3, padding 0 / 1 / 3, dilation 1 / 2, one and two images, the three input views"""
    out, i = [], 0
    for is_2d in (False, True):
        for s in (1, 2, 3):
            for p in (0, 1, 3):
                for d in (1, 2):
                    dst = (F32, F16)[i % 2]
                    view = i % 3
                    n = 1 + (i // 3) % 2
                    if is_2d:
                        case = Im2colCase((3, 2, 3, 5), (11, 9, 3, n), s, 1 + (s % 2), p, (p + 1) % 4, d, 3 - d, True, dst, F16 if dst == F16 else (i // 2) % 2, view, seed=i)
                    else:
                        case = Im2colCase((3, 4, 6, 1), (17, 4, n, 1), s, 0, p, 0, d, 0, False, dst, F16 if dst == F16 else (i // 2) % 2, view, seed=i)
                    out.append(case)
                    i += 1
    # the Whisper front end's own shapes, shortened along the time axis: conv1 (stride 1) and conv2 (stride 2), padding 1, f16 columns
    out.append(Im2colCase((3, 80, 8, 1), (300, 80, 1, 1), 1, 0, 1, 0, 1, 0, False, F16, F16, 0, seed=i))
    out.append(Im2colCase((3, 64, 8, 1), (300, 64, 1, 1), 2, 0, 1, 0, 1, 0, False, F16, F16, 1, seed=i + 1))
    return out


# ------------------------------------------------------------------ the probe
SIGNATURES = {
    "probe_im2col": [C.c_char_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p],
    "probe_mul_mat_f16": [C.c_char_p, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p],
    "probe_conv_1d": [C.c_char_p] + [C.c_int64] * 4 + [C.c_int] * 3 + [C.c_void_p, C.c_void_p],
}


def _lib():
    return probe_lib("conv", "make -C oracle -f whisper.mk whisper", SIGNATURES)


def im2col(dev: str, case: Im2colCase, view: View | None = None, raw: bool = False):
    """IM2COL of `case` on ggml device `dev`: dst contiguous, ggml dims reversed (float32 or float16).  raw: the probe's code"""
    L = _lib()
    v = view or case.view_of_input()
    out = np.zeros(case.ne_dst[::-1], dtype=np.float16 if case.dst_type == F16 else np.float32)
    ne_k, ne_x = np.array(case.ne_kernel, dtype=np.int64), np.array(case.ne_input, dtype=np.int64)
    rc = L.probe_im2col(dev.encode(), case.kernel_type, ne_k.ctypes.data, ne_x.ctypes.data, case.view, case.params.ctypes.data, case.dst_type,
                        ptrs([v.parent]), out.ctypes.data)
    return result(rc, raw, f"probe_im2col({dev}, {case})", out)


def f16_operands(M: int, N: int, K: int, b_view: int, seed: int = 0):
    """a f16 [M, K] and b's parent f16 as mul_mat_f16's probe reads them (b_view 0: [N, K]; 1: [N, K + 8]; 2: [N, K + 3])"""
    rng = np.random.default_rng(12000 + seed)
    a = rng.standard_normal((M, K)).astype(np.float16)
    shape = {0: (N, K), 1: (N, K + 8), 2: (N, K + 3)}[b_view]
    b = (rng.standard_normal(shape) / np.sqrt(K)).astype(np.float16)
    return a, b


def mul_mat_f16(dev: str, M: int, N: int, K: int, b_view: int = 0, operands=None, raw: bool = False):
    """MUL_MAT(a f16 [K, M], b f16 [K, N]) on `dev`: f32 [N, M]"""
    L = _lib()
    a, b = operands if operands is not None else f16_operands(M, N, K, b_view)
    out = np.zeros((N, M), dtype=np.float32)
    rc = L.probe_mul_mat_f16(dev.encode(), M, N, K, b_view, ptrs([a, b]), out.ctypes.data)
    return result(rc, raw, f"probe_mul_mat_f16({dev}, {M}, {N}, {K}, view {b_view})", out)


def mul_mat_f16_reference(a: np.ndarray, b: np.ndarray, b_view: int) -> np.ndarray:
    """the exact products summed in f64: f32 [N, M]"""
    K = a.shape[1]
    return (b[:, :K].astype(np.float64) @ a.astype(np.float64).T).astype(np.float32)


def conv_1d(dev: str, KW: int, IC: int, OC: int, L_: int, s: int, p: int, d: int, seed: int = 0, raw: bool = False):
    """ggml_conv_1d(kernel f16 [OC, IC, KW], x f32 [IC, L]) on `dev`: f32 [OC, OL]"""
    L = _lib()
    rng = np.random.default_rng(13000 + seed)
    k = (rng.standard_normal((OC, IC, KW)) / np.sqrt(IC * KW)).astype(np.float16)
    x = rng.standard_normal((IC, L_)).astype(np.float32)
    out = np.zeros((OC, conv_out(L_, KW, s, p, d)), dtype=np.float32)
    rc = L.probe_conv_1d(dev.encode(), KW, IC, OC, L_, s, p, d, ptrs([k, x]), out.ctypes.data)
    return result(rc, raw, f"probe_conv_1d({dev}, KW={KW} IC={IC} OC={OC} L={L_} s={s} p={p} d={d})", out)
