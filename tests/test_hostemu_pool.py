"""CPU-only: the per-element logic of POOL_2D, UPSCALE, LEAKY_RELU and REPEAT (ggml_b200/csrc/b200_pool.cuh) compiled for the HOST through
tests/hostemu/shim (tests/hostemu/pool_emu.cpp walks dst's elements as ops.cu's kernels do, with the launchers' arguments) and checked
against the reference's own ggml-cpu ops, one-node graphs through oracle/pool_probe.cpp, as raw bits.  The grids:
  POOL_2D     MAX and AVG (a NaN result of AVG equals any NaN: see pool_equal), windows 1-3, strides 1-3, paddings 0-2 (windows wholly in the padding among them), the k2 s1 pool with
              ggml_pool_2d's float padding 0.5, inputs with NaN, +-inf, -0 and equal neighbours, rows padded beyond 4 ne0, two images;
  UPSCALE     integer and fractional factors, a strided and a transposed input;
  LEAKY_RELU  slopes 0.1, 0 and 1 on NaN, +-0 and +-inf (0 x -inf is NaN: a NaN equals any NaN), in place and not, padded rows;
  REPEAT      all five element types ggml-cpu repeats, a strided src, NaN payloads.
The EUNSUPPORTED / EINVAL codes of check_pool_2d, check_upscale, check_leaky_relu and check_repeat (b200_op_checks.h), which the C ABI
launchers and the plug-in's supports_op apply, are pinned here too."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import ggml_b200 as g
from oracle import pool as P

ROOT = Path(__file__).resolve().parents[1]
EMU = ROOT / "tests" / "hostemu"
OK, EUNSUPPORTED, EINVAL = 0, -1, -2
F32, F16, I16, I32, BF16 = P.F32, P.F16, P.I16, P.I32, P.BF16


@pytest.fixture(scope="module")
def emu():
    out = EMU / "_build"
    out.mkdir(exist_ok=True)
    so = out / "libpool_emu.so"
    srcs = [EMU / "pool_emu.cpp", EMU / "shim" / "cuda_shim.h", ROOT / "ggml_b200" / "csrc" / "b200_pool.cuh",
            ROOT / "ggml_b200" / "csrc" / "b200_op_checks.h", ROOT / "include" / "ggml-b200.h"]
    if not so.exists() or so.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", "-mf16c", "-mavx", "-ffp-contract=off", "-Wno-unused-variable",
               f"-I{EMU / 'shim'}", "-o", str(so), str(EMU / "pool_emu.cpp")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(str(so))
    TD = C.POINTER(g.TensorDesc)
    for fn in (L.emu_pool_2d, L.emu_check_pool_2d):
        fn.restype, fn.argtypes = C.c_int, [TD, TD, C.POINTER(g.PoolParams)]
    for fn in (L.emu_upscale, L.emu_check_upscale, L.emu_repeat, L.emu_check_repeat, L.emu_check_leaky_relu):
        fn.restype, fn.argtypes = C.c_int, [TD, TD]
    L.emu_leaky_relu.restype, L.emu_leaky_relu.argtypes = C.c_int, [TD, TD, C.c_float]
    return L


def desc(type_, ne, nb=None, data=4096):
    """a ggml tensor descriptor: ne in ggml order, nb in bytes (packed when None)"""
    d = g.TensorDesc()
    d.data, d.type = data, type_
    ne = tuple(ne) + (1,) * (4 - len(ne))
    nb = nb or P.packed_nb(ne, P.ES[type_])
    for i in range(4):
        d.ne[i], d.nb[i] = ne[i], nb[i]
    return d


def src_desc(src: P.Source, parent: np.ndarray):
    ne, nb = src.view()
    return desc(src.type, ne, nb, parent.ctypes.data + src.offs)


def bits(a):
    return a.view(np.uint32 if a.itemsize == 4 else np.uint16)


def nan_equal(got, want):
    """bit for bit, except that a NaN equals any NaN: which NaN an IEEE operation returns (an AVG window holding NaN or both infinities,
    LEAKY_RELU's 0 x -inf) is the hardware's and the compiler's choice (x86 keeps an operand's or its default NaN, the GPU its canonical one)"""
    nan = np.isnan(got)
    return np.array_equal(nan, np.isnan(want)) and np.array_equal(bits(got)[~nan], bits(want)[~nan])


POOLS, UPSCALES, LEAKIES, REPEATS = P.pool_grid(), P.upscale_grid(), P.leaky_grid(), P.repeat_grid()


def test_grids_cover_the_axes():
    assert {c.op for c in POOLS} == {P.POOL_MAX, P.POOL_AVG} and {c.k0 for c in POOLS} == {1, 2, 3} and {c.s0 for c in POOLS} == {1, 2, 3}
    assert {c.p0 for c in POOLS} >= {0, 1, 2, 0.5} and any(c.p0 >= c.k0 for c in POOLS)          # windows wholly in the padding
    assert any(c.src.parent_ne[0] > c.src.ne[0] for c in POOLS) and any(c.src.ne[3] == 2 for c in POOLS)
    assert any(c.ne_dst[0] != c.src.ne[0] * (c.ne_dst[0] // c.src.ne[0]) for c in UPSCALES) and any(c.src.transpose for c in UPSCALES)
    assert {c.slope for c in LEAKIES} == {0.1, 0.0, 1.0} and any(c.inplace for c in LEAKIES)
    assert {c.src.type for c in REPEATS} == {F32, I32, F16, BF16, I16} and any(c.src.parent_ne != c.src.ne for c in REPEATS)


@pytest.mark.parametrize("case", POOLS, ids=[f"{i}-{c.op}-k{c.k0}{c.k1}-s{c.s0}{c.s1}-p{c.p0}{c.p1}" for i, c in enumerate(POOLS)])
def test_host_compiled_pool_2d_is_bit_identical_to_ggml_cpu(case, emu, ref):
    parent = case.src.parent()
    got = np.zeros(case.ne_dst[::-1], dtype=np.float32)
    p = g.PoolParams(*case.params)
    assert emu.emu_pool_2d(C.byref(src_desc(case.src, parent)), C.byref(desc(F32, case.ne_dst, data=got.ctypes.data)), C.byref(p)) == OK
    want = P.pool_2d("CPU", case, parent)
    assert nan_equal(got, want), (str(case), int((bits(got) != bits(want)).sum()))
    if case.op == P.POOL_MAX:                                  # MAX moves input values: no arithmetic, no NaN result, every bit equal
        assert np.array_equal(bits(got), bits(want)) and not np.isnan(want).any(), str(case)


def test_pool_2d_corner_semantics(emu, ref):
    """a window of padding / NaN / -inf only gives -FLT_MAX under MAX; the float padding 0.5 gives 13 x 13 from 13 x 13"""
    case = P.PoolCase(P.Source(F32, (13, 13, 2, 1)), P.POOL_MAX, 2, 2, 1, 1, 0.5, 0.5)
    assert case.ne_dst == (13, 13, 2, 1)
    parent = np.full((1, 2, 13, 13), np.nan, dtype=np.float32)
    parent[0, 1] = -np.inf
    want = P.pool_2d("CPU", case, parent)
    assert (want == np.finfo(np.float32).min).all()
    corner = P.PoolCase(P.Source(F32, (4, 4, 1, 1)), P.POOL_MAX, 1, 1, 1, 1, 2, 2)              # k 1, p 2: the outer windows are padding
    w = P.pool_2d("CPU", corner, np.ones((1, 1, 4, 4), dtype=np.float32))
    assert w[0, 0, 0, 0] == np.finfo(np.float32).min and w[0, 0, 2, 2] == 1.0


@pytest.mark.parametrize("case", UPSCALES, ids=[str(i) for i in range(len(UPSCALES))])
def test_host_compiled_upscale_is_bit_identical_to_ggml_cpu(case, emu, ref):
    parent = case.src.parent()
    got = np.zeros(tuple(case.ne_dst)[::-1], dtype=np.float32)
    assert emu.emu_upscale(C.byref(src_desc(case.src, parent)), C.byref(desc(F32, case.ne_dst, data=got.ctypes.data))) == OK
    want = P.upscale("CPU", case, parent)
    assert np.array_equal(bits(got), bits(want)), str(case)


@pytest.mark.parametrize("case", LEAKIES, ids=[str(c) for c in LEAKIES])
def test_host_compiled_leaky_relu_is_bit_identical_to_ggml_cpu(case, emu, ref):
    parent = case.src.parent()
    want = P.leaky_relu("CPU", case, parent.copy())
    ne, nb = case.src.view()
    if case.inplace:
        work = parent.copy()
        s = src_desc(case.src, work)
        assert emu.emu_leaky_relu(C.byref(s), C.byref(s), case.slope) == OK
        got = work.reshape(-1)[: want.size]
    else:
        got = np.zeros(ne[::-1], dtype=np.float32)
        assert emu.emu_leaky_relu(C.byref(src_desc(case.src, parent)), C.byref(desc(F32, ne, data=got.ctypes.data)), case.slope) == OK
    assert nan_equal(got, want), str(case)
    ne, nb = case.src.view()
    x = np.lib.stride_tricks.as_strided(parent.reshape(-1)[case.src.offs // 4:], ne[::-1], nb[::-1])
    y = want.reshape(-1)[: x.size].reshape(ne[::-1]) if case.inplace else want
    special = np.isnan(x) | ((x == 0) & np.signbit(x))
    assert special.any() and (bits(y[special]) == 0).all()                                    # NaN and -0 become +0
    assert np.isnan(y).sum() == (np.isneginf(x).sum() if case.slope == 0.0 else 0)            # NaN only from 0 x -inf


@pytest.mark.parametrize("case", REPEATS, ids=[str(c) for c in REPEATS])
def test_host_compiled_repeat_is_bit_identical_to_ggml_cpu(case, emu, ref):
    parent = case.src.parent()
    got = np.zeros(tuple(case.ne_dst)[::-1], dtype=np.uint32 if P.ES[case.src.type] == 4 else np.uint16)
    assert emu.emu_repeat(C.byref(src_desc(case.src, parent)), C.byref(desc(case.src.type, case.ne_dst, data=got.ctypes.data))) == OK
    want = P.repeat("CPU", case, parent)
    assert np.array_equal(got, want.view(got.dtype)), str(case)


# ------------------------------------------------------------------ the checks' codes
def test_check_pool_2d_codes(emu):
    def chk(s, d, *params):
        p = g.PoolParams(*params)
        return emu.emu_check_pool_2d(C.byref(s) if s else None, C.byref(d), C.byref(p))
    x, y = desc(F32, (13, 13, 16, 2)), desc(F32, (6, 6, 16, 2))
    assert chk(x, y, 0, 2, 2, 2, 2, 0, 0) == OK and chk(x, y, 1, 2, 2, 2, 2, 0, 0) == OK
    assert chk(x, y, 2, 2, 2, 2, 2, 0, 0) == EINVAL                                   # POOL_COUNT: ggml-cpu aborts
    assert chk(x, y, -1, 2, 2, 2, 2, 0, 0) == EINVAL
    assert chk(x, y, 0, 0, 2, 2, 2, 0, 0) == EINVAL and chk(x, y, 0, 2, 0, 2, 2, 0, 0) == EINVAL   # window >= 1
    assert chk(x, y, 0, 2, 2, 0, 2, 0, 0) == EINVAL and chk(x, y, 0, 2, 2, 2, 0, 0, 0) == EINVAL   # stride >= 1
    assert chk(x, desc(F32, (6, 6, 8, 2)), 0, 2, 2, 2, 2, 0, 0) == EINVAL                # C differs
    assert chk(x, desc(F32, (6, 6, 16, 1)), 0, 2, 2, 2, 2, 0, 0) == EINVAL               # N differs
    assert chk(x, desc(F32, (13, 13, 16, 2)), 0, 2, 2, 1, 1, 0, 0) == OK                 # OW / OH are dst's own (float paddings)
    assert chk(desc(F16, (13, 13, 16, 2)), y, 0, 2, 2, 2, 2, 0, 0) == EUNSUPPORTED       # f16 input
    assert chk(x, desc(F16, (6, 6, 16, 2)), 0, 2, 2, 2, 2, 0, 0) == EUNSUPPORTED
    assert chk(desc(F32, (13, 13, 16, 2), (8, 104, 1352, 21632)), y, 0, 2, 2, 2, 2, 0, 0) == EUNSUPPORTED    # src nb0 != 4
    assert chk(desc(F32, (13, 13, 16, 2), (4, 64, 1000, 16000)), y, 0, 2, 2, 2, 2, 0, 0) == OK              # any other src strides
    assert chk(x, desc(F32, (6, 6, 16, 2), (4, 28, 168, 2688)), 0, 2, 2, 2, 2, 0, 0) == EUNSUPPORTED        # dst not packed
    assert chk(None, y, 0, 2, 2, 2, 2, 0, 0) == EUNSUPPORTED
    assert chk(desc(F32, (13, 13, 0, 2)), desc(F32, (6, 6, 0, 2)), 0, 2, 2, 2, 2, 0, 0) == OK             # empty


def test_check_upscale_codes(emu):
    chk = lambda s, d: emu.emu_check_upscale(C.byref(s) if s else None, C.byref(d))
    x = desc(F32, (13, 13, 128, 1))
    assert chk(x, desc(F32, (26, 26, 128, 1))) == OK and chk(x, desc(F32, (13, 13, 128, 1))) == OK
    assert chk(desc(F32, (2, 5, 7, 11)), desc(F32, (5, 7, 11, 13))) == OK                 # fractional factors
    assert chk(x, desc(F32, (12, 26, 128, 1))) == EINVAL and chk(x, desc(F32, (26, 26, 64, 1))) == EINVAL   # dst smaller than src
    assert chk(desc(F32, (0, 13, 128, 1)), desc(F32, (26, 26, 128, 1))) == EINVAL         # empty src, non-empty dst
    assert chk(desc(F32, (0, 13, 128, 1)), desc(F32, (0, 26, 128, 1))) == OK
    assert chk(desc(F16, (13, 13, 128, 1)), desc(F16, (26, 26, 128, 1))) == EUNSUPPORTED and chk(x, desc(F16, (26, 26, 128, 1))) == EUNSUPPORTED
    assert chk(desc(F32, (13, 13, 128, 1), (52, 4, 676, 86528)), desc(F32, (26, 26, 128, 1))) == OK         # transposed src
    assert chk(None, desc(F32, (26, 26, 128, 1))) == EUNSUPPORTED


def test_check_leaky_relu_codes(emu):
    chk = lambda s, d: emu.emu_check_leaky_relu(C.byref(s) if s else None, C.byref(d))
    x = desc(F32, (10, 5, 4, 3))
    assert chk(x, x) == OK and chk(x, desc(F32, (10, 5, 4, 3))) == OK
    assert chk(x, desc(F32, (10, 5, 4, 2))) == EINVAL                                     # shapes differ
    assert chk(desc(F16, (10, 5, 4, 3)), desc(F16, (10, 5, 4, 3))) == EUNSUPPORTED
    assert chk(desc(F32, (10, 5, 4, 3), (20, 200, 1000, 4000)), x) == EUNSUPPORTED         # src nb0 != 4
    assert chk(x, desc(F32, (10, 5, 4, 3), (20, 200, 1000, 4000))) == EUNSUPPORTED
    assert chk(desc(F32, (10, 5, 4, 3), (4, 60, 300, 1200)), x) == OK                      # padded rows
    assert chk(None, x) == EUNSUPPORTED


def test_check_repeat_codes(emu):
    chk = lambda s, d: emu.emu_check_repeat(C.byref(s) if s else None, C.byref(d))
    for t in (F32, I32, F16, BF16, I16):
        assert chk(desc(t, (1, 1, 16, 1)), desc(t, (13, 13, 16, 2))) == OK
    assert chk(desc(8, (32, 1), (34, 34, 34, 34)), desc(8, (32, 4), (34, 34, 136, 136))) == EUNSUPPORTED                         # Q8_0: ggml-cpu aborts
    assert chk(desc(F32, (1, 1, 16, 1)), desc(F16, (13, 13, 16, 2))) == EUNSUPPORTED       # types differ
    assert chk(desc(F32, (1, 1, 16, 1)), desc(F32, (13, 13, 24, 2))) == EINVAL             # 24 % 16
    assert chk(desc(F32, (3, 2, 4, 1)), desc(F32, (7, 4, 8, 2))) == EINVAL
    assert chk(desc(F32, (0, 1, 16, 1)), desc(F32, (13, 13, 16, 2))) == EINVAL             # an empty src repeats into an empty dst only
    assert chk(desc(F32, (0, 1, 16, 1)), desc(F32, (0, 13, 16, 2))) == OK
    assert chk(desc(F32, (3, 2, 4, 1), (8, 24, 48, 192)), desc(F32, (6, 4, 8, 2))) == EUNSUPPORTED           # src nb0 != 4
    assert chk(desc(F32, (3, 2, 4, 1)), desc(F32, (6, 4, 8, 2), (8, 48, 192, 1536))) == EUNSUPPORTED         # dst nb0 != 4
    assert chk(desc(F16, (3, 2, 4, 1), (2, 10, 40, 160)), desc(F16, (6, 4, 8, 2))) == OK                     # any other src strides
    assert chk(None, desc(F32, (6, 4, 8, 2))) == EUNSUPPORTED
