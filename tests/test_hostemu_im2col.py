"""CPU-only: the per-element logic of IM2COL (ggml_b200/csrc/b200_conv.cuh) compiled for the HOST through tests/hostemu/shim
(tests/hostemu/conv_emu.cpp walks dst's elements as ops.cu's im2col_kernel does) and checked against the reference's own ggml-cpu op,
one-node graphs through oracle/conv_probe.cpp.  Both dst types must be BIT-IDENTICAL to ggml-cpu: f32 columns are copies, f16 columns
are rounded once by __float2half_rn, which rounds as F16C does.  The grid covers 1-D and 2-D, f32 and f16 dst, strides 1 / 2 / 3, padding
0 / 1 / 3, dilation 1 / 2, one and two images, inputs with spread channel / image strides and with spread rows (which ggml-cpu reads as
packed), values that round to fp16 ties, subnormals and infinity, and the Whisper front end's two conv shapes.

check_im2col (b200_op_checks.h), which both ggml_b200_op_im2col and the plug-in's supports_op apply, is pinned here too, with the f16 x f16
form of check_mul_mat_f."""
import ctypes as C

import numpy as np
import pytest

import ggml_b200 as g
from hostemu.emu import EINVAL, EUNSUPPORTED, OK, desc, load
from oracle import conv as V

F32, F16 = 0, 1


@pytest.fixture(scope="module")
def emu():
    L = load("conv_emu")
    L.emu_im2col.restype = C.c_int
    L.emu_im2col.argtypes = [C.POINTER(g.TensorDesc)] * 3 + [C.POINTER(g.Im2colParams)]
    return L


@pytest.fixture(scope="module")
def checks():
    L = load("op_checks_emu")
    L.emu_check_im2col.restype = C.c_int
    L.emu_check_im2col.argtypes = [C.POINTER(g.TensorDesc)] * 3 + [C.POINTER(g.Im2colParams)]
    L.emu_check_mul_mat_f.restype = C.c_int
    L.emu_check_mul_mat_f.argtypes = [C.POINTER(g.TensorDesc)] * 3
    return L


def params(case: V.Im2colCase) -> g.Im2colParams:
    return g.Im2colParams(*[int(v) for v in case.params])


def emu_im2col(L, case: V.Im2colCase, view):
    out = np.zeros(case.ne_dst[::-1], dtype=np.float16 if case.dst_type == F16 else np.float32)
    k = desc(case.kernel_type, case.ne_kernel)
    x = desc(F32, view.ne, view.nb, view.parent.ctypes.data + view.offs)
    d = desc(case.dst_type, case.ne_dst, data=out.ctypes.data)
    rc = L.emu_im2col(C.byref(k), C.byref(x), C.byref(d), C.byref(params(case)))
    assert rc == OK, (str(case), rc)
    return out


GRID = V.im2col_grid()


def test_im2col_grid_covers_the_axes():
    assert {c.is_2d for c in GRID} == {False, True} and {c.dst_type for c in GRID} == {F32, F16} and {c.view for c in GRID} == {0, 1, 2}
    assert {c.s0 for c in GRID} == {1, 2, 3} and {c.p0 for c in GRID} == {0, 1, 3} and {c.d0 for c in GRID} == {1, 2}
    assert {(c.ne_input[3] if c.is_2d else c.ne_input[2]) for c in GRID} == {1, 2}
    assert {c.kernel_type for c in GRID if c.dst_type == F32} == {F32, F16}


@pytest.mark.parametrize("case", GRID, ids=[f"{i}-{'2d' if c.is_2d else '1d'}-s{c.s0}p{c.p0}d{c.d0}-v{c.view}-{'f16' if c.dst_type else 'f32'}"
                                            for i, c in enumerate(GRID)])
def test_host_compiled_im2col_is_bit_identical_to_ggml_cpu(case, emu, ref):
    view = case.view_of_input()
    got = emu_im2col(emu, case, view)
    want = V.im2col("CPU", case, view)
    u = np.uint16 if case.dst_type == F16 else np.uint32
    assert got.shape == want.shape and np.array_equal(got.view(u), want.view(u)), (str(case), int((got.view(u) != want.view(u)).sum()))


def test_check_im2col_codes(checks):
    def chk(k, x, d, p):
        return checks.emu_check_im2col(C.byref(k), C.byref(x), C.byref(d), C.byref(p)) if k is not None else \
            checks.emu_check_im2col(None, C.byref(x), C.byref(d), C.byref(p))
    P = lambda s0=1, s1=0, p0=1, p1=0, d0=1, d1=0, two=0: g.Im2colParams(s0, s1, p0, p1, d0, d1, two)
    k, x = desc(F16, (3, 4, 6)), desc(F32, (17, 4, 2))
    d16, d32 = desc(F16, (12, 17, 2)), desc(F32, (12, 17, 2))
    assert chk(k, x, d16, P()) == OK and chk(k, x, d32, P()) == OK
    assert chk(desc(F32, (3, 4, 6)), x, d32, P()) == OK                                        # f32 kernel, f32 columns
    assert chk(desc(F32, (3, 4, 6)), x, d16, P()) == EUNSUPPORTED                              # f16 columns need an f16 kernel
    assert chk(k, x, d16, P(two=2)) == EINVAL                                                  # is_2D 0 or 1
    assert chk(k, x, d16, P(s0=0)) == EINVAL and chk(k, x, d16, P(d0=0)) == EINVAL             # s, d >= 1
    assert chk(k, x, d16, P(s1=-1, d1=-3)) == OK                                               # s1 / d1 unused in 1-D
    assert chk(None, x, d16, P()) == EUNSUPPORTED
    assert chk(k, desc(F16, (17, 4, 2)), d16, P()) == EUNSUPPORTED                             # f32 input only
    assert chk(k, desc(F32, (17, 4, 2), (8, 136, 544, 1088)), d16, P()) == EUNSUPPORTED        # input nb0 != 4
    assert chk(k, desc(F32, (17, 4, 2), (4, 100, 1000, 2000)), d16, P()) == OK                 # any other input strides
    assert chk(k, x, desc(F16, (12, 17, 2), (2, 26, 17 * 26, 2 * 17 * 26)), P()) == EUNSUPPORTED   # dst not packed
    assert chk(k, x, desc(F16, (12, 16, 2)), P()) == EUNSUPPORTED                               # OW
    assert chk(k, x, desc(F16, (12, 17, 2)), P(p0=0)) == EUNSUPPORTED                           # OW of the params: 15
    assert chk(k, x, desc(F16, (12, 15, 2)), P(p0=0)) == OK
    assert chk(k, x, desc(F16, (12, 9, 2)), P(s0=2)) == OK                                     # (17 + 2 - 2 - 1) / 2 + 1
    assert chk(k, x, desc(F16, (12, 17, 2)), P(d0=2)) == EUNSUPPORTED and chk(k, x, desc(F16, (12, 15, 2)), P(d0=2)) == OK
    assert chk(k, desc(F32, (17, 4, 2, 2)), desc(F16, (12, 17, 2, 2)), P()) == EUNSUPPORTED    # the 1-D input is 3-D
    assert chk(k, desc(F32, (17, 5, 2)), d16, P()) == EUNSUPPORTED                              # IC KW
    assert chk(k, desc(F32, (17, 4, 0)), desc(F16, (12, 17, 0)), P()) == OK                     # empty
    big = desc(F32, (17, 4, 2), (4, 1 << 31, 1 << 32, 1 << 33))                                 # channel offsets beyond an int
    assert chk(k, big, d16, P()) == EUNSUPPORTED
    assert chk(k, desc(F32, (17, 4, 2), (4, 68, (1 << 31) - 4, 1 << 33)), d16, P()) == OK
    # 2-D: kernel [KW, KH, IC, OC], input [IW, IH, IC, N], dst [IC KH KW, OW, OH, N]
    k2, x2 = desc(F16, (3, 2, 3, 5)), desc(F32, (11, 9, 3, 2))
    P2 = lambda **kw: P(**{"s1": 1, "p1": 0, "d1": 1, "p0": 0, "two": 1, **kw})
    assert chk(k2, x2, desc(F32, (18, 9, 8, 2)), P2()) == OK
    assert chk(k2, x2, desc(F32, (18, 9, 8, 2)), P2(s1=0)) == EINVAL and chk(k2, x2, desc(F32, (18, 9, 8, 2)), P2(d1=0)) == EINVAL
    assert chk(k2, x2, desc(F32, (18, 9, 4, 2)), P2(s1=2)) == OK
    assert chk(k2, x2, desc(F32, (18, 9, 8, 1)), P2()) == EUNSUPPORTED                          # N
    assert chk(k2, desc(F32, (11, 9, 3, 2), (4, 44, 1 << 31, 1 << 33)), desc(F32, (18, 9, 8, 2)), P2()) == EUNSUPPORTED   # channel stride
    assert chk(k2, desc(F32, (11, 9, 3, 2), (4, 60, 600, 1800)), desc(F32, (18, 9, 8, 2)), P2()) == OK                    # rows spread


def test_check_mul_mat_f_takes_f16_src1_with_f16_src0_only(checks):
    chk = lambda a, b, d: checks.emu_check_mul_mat_f(C.byref(a), C.byref(b), C.byref(d))
    assert chk(desc(F16, (64, 16)), desc(F16, (64, 9)), desc(F32, (16, 9))) == OK
    assert chk(desc(F16, (64, 16)), desc(F32, (64, 9)), desc(F32, (16, 9))) == OK
    assert chk(desc(F32, (64, 16)), desc(F16, (64, 9)), desc(F32, (16, 9))) == EUNSUPPORTED
    assert chk(desc(F16, (64, 16)), desc(F16, (64, 9)), desc(F16, (16, 9))) == EUNSUPPORTED
    assert chk(desc(F16, (64, 16, 2)), desc(F16, (64, 9, 6)), desc(F32, (16, 9, 6))) == OK      # batch broadcast
    assert chk(desc(F16, (64, 16, 4)), desc(F16, (64, 9, 6)), desc(F32, (16, 9, 6))) == EUNSUPPORTED
