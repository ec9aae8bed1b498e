"""CPU-only: the per-row / per-element logic of WIN_PART, WIN_UNPART, GET_REL_POS, ADD_REL_POS and CONV_TRANSPOSE_2D (ggml_b200/csrc/b200_sam.cuh)
compiled for the HOST through tests/hostemu/shim (tests/hostemu/sam_emu.cpp walks dst as ops.cu's kernels do, with the launchers' arguments)
and checked against the reference's own ggml-cpu ops, one-node graphs through oracle/sam_probe.cpp.  The grids:
  WIN_PART / WIN_UNPART  windows that divide the image and ones that do not, w = 1, a window larger than the image, the SAM window 14 on a
                         padded image, more windows than the image needs; raw bits (NaN payloads, +-inf, -0 kept);
  GET_REL_POS            w = 1 .. 64, raw f16 words;
  ADD_REL_POS            L = 1, 2, 7, 14, square and non-square query grids, in place and out of place, values for which the two orders of
                         the adds round differently: bit for bit, and the order is pinned against a numpy restatement of both orders;
  CONV_TRANSPOSE_2D      s < K, s = K, s > K, Cin = 1, Cin / Cout not multiples of the device tile, strided operands, NaN / +-inf / -0
                         inputs: within NMSE 1e-10 of ggml-cpu and of an f64 reference on the fp16-rounded operands;
  SIN / COS              ggml-cpu (glibc sinf / cosf) within 1 ulp of the f64 value, the bound the device's 2 ulp is set against.
The EUNSUPPORTED / EINVAL codes of the five checks (b200_op_checks.h), which the C ABI launchers and the plug-in's supports_op apply, are
pinned here too."""
import ctypes as C

import numpy as np
import pytest

import ggml_b200 as g
from hostemu.emu import EINVAL, EUNSUPPORTED, OK, bits, desc, load, view_desc
from oracle import oracle as O
from oracle import pool as P
from oracle import sam as S

F32, F16, BF16 = P.F32, P.F16, P.BF16
CONV_NMSE = 1e-10


def signatures(L, prefix):
    """the ctypes signatures of the five ops' entries <prefix><op>: the emus (emu_) and their checks (emu_check_) take the same arguments"""
    TD = C.POINTER(g.TensorDesc)
    for op, args in (("win_part", [TD, TD, C.c_int32, C.c_int32, C.c_int32]), ("win_unpart", [TD, TD, C.c_int32]), ("get_rel_pos", [TD, TD]),
                     ("add_rel_pos", [TD] * 4), ("conv_transpose_2d", [TD] * 3 + [C.c_int32])):
        fn = getattr(L, prefix + op)
        fn.restype, fn.argtypes = C.c_int, args
    return L


@pytest.fixture(scope="module")
def emu():
    return signatures(load("sam_emu"), "emu_")


@pytest.fixture(scope="module")
def checks():
    return signatures(load("op_checks_emu"), "emu_check_")


WIN_PARTS, WIN_UNPARTS, RELPOS, ADDS, CONVS = S.win_part_grid(), S.win_unpart_grid(), S.rel_pos_grid(), S.add_rel_pos_grid(), S.conv_transpose_grid()


def test_grids_cover_the_axes():
    assert any(c.src.ne[1] % c.w for c in WIN_PARTS) and any(c.src.ne[1] % c.w == 0 and c.src.ne[2] % c.w == 0 for c in WIN_PARTS)
    assert any(c.w == 1 for c in WIN_PARTS) and any(c.w > c.src.ne[1] for c in WIN_PARTS)
    assert any(c.src.ne[3] > S.cdiv(c.w0, c.w) * S.cdiv(c.h0, c.w) for c in WIN_UNPARTS)
    assert [c.w for c in RELPOS] == list(range(1, 65))
    assert {c.L for c in ADDS} == {1, 2, 7, 14} and {c.inplace for c in ADDS} == {False, True} and any(c.A != c.B for c in ADDS)
    assert any(c.s < c.Kw for c in CONVS) and any(c.s == c.Kw for c in CONVS) and any(c.s > c.Kw for c in CONVS)
    assert any(c.Cin == 1 for c in CONVS) and any(c.Cin % 32 and c.Cin > 32 for c in CONVS) and any(c.Cout % 32 and c.Cout > 32 for c in CONVS)
    assert any(c.specials for c in CONVS) and any(c.k_parent_ne and c.x_parent_ne for c in CONVS)


@pytest.mark.parametrize("case", WIN_PARTS, ids=[str(c) for c in WIN_PARTS])
def test_host_compiled_win_part_is_bit_identical_to_ggml_cpu(case, emu, ref):
    parent = case.src.parent()
    got = np.full(case.ne_dst[::-1], 0xdeadbeef, dtype=np.uint32)
    npx, npy = S.cdiv(case.src.ne[1], case.w), S.cdiv(case.src.ne[2], case.w)
    assert emu.emu_win_part(C.byref(view_desc(case.src, parent)), C.byref(desc(F32, case.ne_dst, data=got.ctypes.data)), npx, npy, case.w) == OK
    want = S.win_part("CPU", case, parent)
    assert np.array_equal(got, want), str(case)
    assert np.isnan(parent).any() and (want == 0x80000000).any()              # NaN and -0 words among the moved ones


@pytest.mark.parametrize("case", WIN_UNPARTS, ids=[str(c) for c in WIN_UNPARTS])
def test_host_compiled_win_unpart_is_bit_identical_to_ggml_cpu(case, emu, ref):
    parent = case.src.parent()
    got = np.full(case.ne_dst[::-1], 0xdeadbeef, dtype=np.uint32)
    assert emu.emu_win_unpart(C.byref(view_desc(case.src, parent)), C.byref(desc(F32, case.ne_dst, data=got.ctypes.data)), case.w) == OK
    assert np.array_equal(got, S.win_unpart("CPU", case, parent)), str(case)


def test_win_unpart_inverts_win_part(ref):
    part = S.WinPartCase(P.Source(F32, (5, 9, 7, 1), seed=7), 4)
    parent = part.src.parent()
    windows = S.win_part("CPU", part, parent)
    back = S.win_unpart("CPU", S.WinUnpartCase(P.Source(F32, part.ne_dst), 9, 7, 4), windows.view(np.float32).copy())
    assert np.array_equal(back.reshape(-1), parent.view(np.uint32).reshape(-1))


@pytest.mark.parametrize("case", RELPOS, ids=[f"w{c.w}" for c in RELPOS])
def test_host_compiled_get_rel_pos_is_bit_identical_to_ggml_cpu(case, emu, ref):
    parent = case.src.parent()
    got = np.full(case.ne_dst[::-1], 0xdead, dtype=np.uint16)
    assert emu.emu_get_rel_pos(C.byref(view_desc(case.src, parent)), C.byref(desc(F16, case.ne_dst, data=got.ctypes.data))) == OK
    want = S.get_rel_pos("CPU", case, parent)
    assert np.array_equal(got, want), str(case)
    w, rows = case.w, parent.reshape(2 * case.w - 1, -1)
    assert np.array_equal(want.reshape(w, w, -1), np.stack([np.stack([rows[(w - 1 - i1) + i2] for i1 in range(w)]) for i2 in range(w)]))


@pytest.mark.parametrize("case", ADDS, ids=[str(c) for c in ADDS])
def test_host_compiled_add_rel_pos_is_bit_identical_to_ggml_cpu(case, emu, ref):
    a, pw, ph = case.parents()
    want = S.add_rel_pos("CPU", case, (a.copy(), pw, ph))
    sa, sw, sh = case.sources()
    if case.inplace:
        got = a.copy()
        d = view_desc(sa, got)
        assert emu.emu_add_rel_pos(C.byref(d), C.byref(view_desc(sw, pw)), C.byref(view_desc(sh, ph)), C.byref(d)) == OK
    else:
        got = np.zeros(case.ne_dst[::-1], dtype=np.float32)
        assert emu.emu_add_rel_pos(C.byref(view_desc(sa, a)), C.byref(view_desc(sw, pw)), C.byref(view_desc(sh, ph)),
                                   C.byref(desc(F32, case.ne_dst, data=got.ctypes.data))) == OK
    nan = np.isnan(want)
    assert np.array_equal(nan, np.isnan(got)) and np.array_equal(bits(got)[~nan], bits(want)[~nan]), str(case)
    # ggml-cpu's order of the two adds, restated: ph first where kh <= kw, pw first elsewhere
    ggml = S.add_rel_pos_numpy(a[0], pw, ph, case.L)
    assert np.array_equal(bits(ggml)[~nan[0]], bits(want[0])[~nan[0]])
    # the values make the orders differ: pw first differs somewhere (kh <= kw takes ph first), and for L >= 2 so does ph first everywhere
    for order in ("pw", "ph") if case.L >= 2 else ("pw",):
        other = S.add_rel_pos_numpy(a[0], pw, ph, case.L, order)
        assert not np.array_equal(bits(other)[~nan[0]], bits(want[0])[~nan[0]]), (str(case), order)


def conv_emu(emu, case, k, x):
    ks, xs = case.sources()
    got = np.zeros(case.ne_dst[::-1], dtype=np.float32)
    rc = emu.emu_conv_transpose_2d(C.byref(view_desc(ks, k)), C.byref(view_desc(xs, x)), C.byref(desc(F32, case.ne_dst, data=got.ctypes.data)), case.s)
    return rc, got


def finite_nmse(got, want):
    """NMSE over the elements where want is finite, after the NaN and +-inf positions (and the infinities' signs) are found equal"""
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isposinf(got), np.isposinf(want))
    assert np.array_equal(np.isneginf(got), np.isneginf(want))
    f = np.isfinite(want)
    return O.nmse(got[f].astype(np.float64), want[f].astype(np.float64))


@pytest.mark.parametrize("case", CONVS, ids=[str(c) for c in CONVS])
def test_host_compiled_conv_transpose_2d_is_within_the_gate(case, emu, ref):
    k, x = case.parents()
    rc, got = conv_emu(emu, case, k, x)
    assert rc == OK
    want = S.conv_transpose_2d("CPU", case, (k, x))
    assert finite_nmse(got, want) <= CONV_NMSE, str(case)
    exact = S.conv_transpose_2d_reference(case, k, x)
    assert finite_nmse(got[0], exact) <= CONV_NMSE, str(case)
    if case.specials:
        assert np.isnan(want).any() and np.isinf(want).any()


def test_conv_transpose_2d_adds_taps_in_ggml_cpu_order(emu, ref):
    """Cin = 1: every tap's dot is one exact product, so only the order of the taps decides the bits, and ggml-cpu's order (ascending input
    row, then column, from +0.0) is the header's: bit-identical, although a different order gives different bits"""
    case = S.ConvT2dCase(1, 4, 3, 3, 9, 8, 1, seed=30)
    k, x = case.parents()
    x *= np.exp2(np.random.default_rng(31).integers(-10, 10, x.shape)).astype(np.float32)
    rc, got = conv_emu(emu, case, k, x)
    want = S.conv_transpose_2d("CPU", case, (k, x))
    assert rc == OK and np.array_equal(bits(got), bits(want))
    rev = np.zeros_like(want[0])
    xx = x[0, 0].astype(np.float16).astype(np.float32)
    for iy in reversed(range(case.H)):
        for ix in reversed(range(case.W)):
            rev[:, iy: iy + 3, ix: ix + 3] += xx[iy, ix] * k[0, :, :, :].astype(np.float32)
    assert not np.array_equal(bits(rev), bits(want[0]))


@pytest.mark.parametrize("case", S.sin_cos_grid(), ids=["sin", "cos"])
def test_ggml_cpu_sin_cos_are_within_one_ulp(case, ref):
    """the CPU side of the device's 2-ulp gate: glibc's sinf / cosf, as ggml-cpu calls them, against the f64 value"""
    x = S.sin_cos_parent(case)
    want = S.sin_cos("CPU", case, x)
    ref64 = (np.sin if case.op == S.SIN else np.cos)(x.astype(np.float64))
    fin = np.isfinite(ref64)
    assert np.array_equal(np.isnan(want), ~fin)
    assert S.ulp_error(want[fin], ref64[fin]).max() <= 1.0
    if case.op == S.SIN:
        z = (x == 0)
        assert np.array_equal(np.signbit(want[z]), np.signbit(x[z]))


# ------------------------------------------------------------------ the checks' codes
def test_check_win_part_codes(checks):
    chk = lambda s, d, npx, npy, w: checks.emu_check_win_part(C.byref(s) if s else None, C.byref(d), npx, npy, w)
    x = desc(F32, (768, 64, 64, 1))
    assert chk(x, desc(F32, (768, 14, 14, 25)), 5, 5, 14) == OK
    assert chk(desc(F32, (6, 32, 32, 1)), desc(F32, (6, 14, 14, 9)), 3, 3, 14) == OK
    assert chk(x, desc(F32, (768, 14, 14, 25)), 4, 5, 14) == EINVAL                    # npx != ceil(W0 / w)
    assert chk(x, desc(F32, (768, 14, 14, 25)), 5, 6, 14) == EINVAL
    assert chk(x, desc(F32, (768, 14, 14, 24)), 5, 5, 14) == EINVAL                    # dst extents
    assert chk(x, desc(F32, (768, 14, 13, 25)), 5, 5, 14) == EINVAL
    assert chk(x, desc(F32, (768, 14, 14, 25)), 5, 5, 0) == EINVAL                     # w < 1
    assert chk(desc(F32, (768, 64, 64, 2)), desc(F32, (768, 14, 14, 25)), 5, 5, 14) == EINVAL
    assert chk(desc(F16, (768, 64, 64, 1)), desc(F16, (768, 14, 14, 25)), 5, 5, 14) == EUNSUPPORTED
    assert chk(desc(F32, (768, 64, 64, 1), (4, 4096, 4096 * 64, 4096 * 4096)), desc(F32, (768, 14, 14, 25)), 5, 5, 14) == EUNSUPPORTED  # not packed
    assert chk(x, desc(F32, (768, 14, 14, 25), (4, 3200, 3200 * 14, 3200 * 196)), 5, 5, 14) == EUNSUPPORTED
    assert chk(None, desc(F32, (768, 14, 14, 25)), 5, 5, 14) == EUNSUPPORTED
    assert chk(desc(F32, (0, 64, 64, 1)), desc(F32, (0, 14, 14, 25)), 5, 5, 14) == OK   # empty


def test_check_win_unpart_codes(checks):
    chk = lambda s, d, w: checks.emu_check_win_unpart(C.byref(s) if s else None, C.byref(d), w)
    y = desc(F32, (768, 64, 64, 1))
    assert chk(desc(F32, (768, 14, 14, 25)), y, 14) == OK and chk(desc(F32, (768, 14, 14, 26)), y, 14) == OK
    assert chk(desc(F32, (768, 14, 14, 24)), y, 14) == EINVAL                          # the reads would leave src
    assert chk(desc(F32, (768, 14, 14, 25)), y, 13) == EINVAL and chk(desc(F32, (768, 14, 14, 25)), y, 0) == EINVAL
    assert chk(desc(F32, (768, 14, 14, 25)), desc(F32, (512, 64, 64, 1)), 14) == EINVAL
    assert chk(desc(F16, (768, 14, 14, 25)), desc(F16, (768, 64, 64, 1)), 14) == EUNSUPPORTED
    assert chk(desc(F32, (768, 14, 14, 25), (4, 4096, 4096 * 14, 4096 * 196)), y, 14) == EUNSUPPORTED
    assert chk(None, y, 14) == EUNSUPPORTED


def test_check_get_rel_pos_codes(checks):
    chk = lambda s, d: checks.emu_check_get_rel_pos(C.byref(s) if s else None, C.byref(d))
    assert chk(desc(F16, (64, 127)), desc(F16, (64, 64, 64))) == OK and chk(desc(F16, (3, 1)), desc(F16, (3, 1, 1))) == OK
    assert chk(desc(F16, (64, 125)), desc(F16, (64, 64, 64))) == EINVAL                # 2w - 1 rows
    assert chk(desc(F16, (64, 127)), desc(F16, (64, 64, 63))) == EINVAL and chk(desc(F16, (64, 127)), desc(F16, (32, 64, 64))) == EINVAL
    assert chk(desc(BF16, (64, 127)), desc(F16, (64, 64, 64))) == EUNSUPPORTED         # ggml-cpu writes BF16 bits into F16: declined
    assert chk(desc(F32, (64, 127)), desc(F32, (64, 64, 64))) == EUNSUPPORTED
    assert chk(desc(F16, (64, 127), (2, 256, 256 * 127, 256 * 127)), desc(F16, (64, 64, 64))) == EUNSUPPORTED   # padded rows
    assert chk(None, desc(F16, (64, 64, 64))) == EUNSUPPORTED


def test_check_add_rel_pos_codes(checks):
    chk = lambda a, w, h, d: checks.emu_check_add_rel_pos(*(C.byref(t) if t else None for t in (a, w, h, d)))
    a, p = desc(F32, (4096, 4096, 12, 1)), desc(F32, (64, 64, 64, 12))
    assert chk(a, p, p, a) == OK and chk(desc(F32, (196, 196, 300)), desc(F32, (14, 14, 14, 300)), desc(F32, (14, 14, 14, 300)), desc(F32, (196, 196, 300))) == OK
    assert chk(a, p, desc(F32, (64, 64, 64, 11)), a) == EINVAL                         # pw and ph differ
    assert chk(a, p, p, desc(F32, (4096, 4096, 11, 1))) == EINVAL                       # dst differs
    assert chk(desc(F32, (4095, 4096, 12, 1)), p, p, desc(F32, (4095, 4096, 12, 1))) == EINVAL   # L L
    assert chk(desc(F32, (4096, 4095, 12, 1)), p, p, desc(F32, (4096, 4095, 12, 1))) == EINVAL   # A B
    assert chk(desc(F32, (4096, 4096, 11, 1)), p, p, desc(F32, (4096, 4096, 11, 1))) == EINVAL   # P
    assert chk(desc(F32, (4096, 4096, 12, 2)), p, p, desc(F32, (4096, 4096, 12, 2))) == EUNSUPPORTED   # ne3 > 1: ggml-cpu adds to the first slice
    assert chk(desc(F16, (4096, 4096, 12, 1)), p, p, desc(F16, (4096, 4096, 12, 1))) == EUNSUPPORTED
    assert chk(a, desc(F32, (64, 64, 64, 12), (4, 512, 512 * 64, 512 * 4096)), p, a) == EUNSUPPORTED  # not packed
    assert chk(None, p, p, a) == EUNSUPPORTED and chk(a, p, None, a) == EUNSUPPORTED


def test_check_conv_transpose_2d_codes(checks):
    chk = lambda k, x, d, s: checks.emu_check_conv_transpose_2d(*(C.byref(t) if t else None for t in (k, x, d)), s)
    k, x = desc(F16, (2, 2, 64, 256)), desc(F32, (64, 64, 256, 1))
    assert chk(k, x, desc(F32, (128, 128, 64, 1)), 2) == OK
    assert chk(desc(F16, (3, 3, 4, 5)), desc(F32, (6, 5, 5, 1)), desc(F32, (8, 7, 4, 1)), 1) == OK
    assert chk(k, x, desc(F32, (128, 128, 64, 1)), 0) == EINVAL                        # stride < 1
    assert chk(k, x, desc(F32, (127, 128, 64, 1)), 2) == EINVAL and chk(k, x, desc(F32, (128, 129, 64, 1)), 2) == EINVAL
    assert chk(k, x, desc(F32, (128, 128, 32, 1)), 2) == EINVAL                        # Cout
    assert chk(k, desc(F32, (64, 64, 128, 1)), desc(F32, (128, 128, 64, 1)), 2) == EINVAL   # Cin
    assert chk(k, desc(F32, (64, 64, 256, 2)), desc(F32, (128, 128, 64, 2)), 2) == EUNSUPPORTED   # a batch
    assert chk(desc(F32, (2, 2, 64, 256)), x, desc(F32, (128, 128, 64, 1)), 2) == EUNSUPPORTED   # f32 kernel
    assert chk(k, desc(F16, (64, 64, 256, 1)), desc(F32, (128, 128, 64, 1)), 2) == EUNSUPPORTED
    assert chk(desc(F16, (2, 2, 64, 256), (2, 6, 12, 768)), x, desc(F32, (128, 128, 64, 1)), 2) == EUNSUPPORTED  # kernel rows padded
    assert chk(desc(F16, (2, 2, 64, 256), (2, 4, 16, 1024)), x, desc(F32, (128, 128, 64, 1)), 2) == OK        # padded planes
    assert chk(k, desc(F32, (64, 64, 256, 1), (4, 512, 512 * 64, 512 * 64 * 256)), desc(F32, (128, 128, 64, 1)), 2) == OK   # padded rows
    assert chk(k, desc(F32, (64, 64, 256, 1), (8, 512, 512 * 64, 512 * 64 * 256)), desc(F32, (128, 128, 64, 1)), 2) == EUNSUPPORTED
    assert chk(k, x, desc(F32, (128, 128, 64, 1), (4, 1024, 1024 * 128, 1024 * 128 * 64)), 2) == EUNSUPPORTED   # dst not packed
    assert chk(desc(F16, (1, 1, 4, 4)), desc(F32, (4, 4, 4, 1)), desc(F32, (1021, 1021, 4, 1)), 340) == EUNSUPPORTED   # s > 255
    assert chk(None, x, desc(F32, (128, 128, 64, 1)), 2) == EUNSUPPORTED
