"""CPU-only: the per-element logic of the training ops (ggml_b200/csrc/b200_train.cuh) compiled for the HOST through tests/hostemu/shim
(tests/hostemu/train_emu.cpp drives it as ops.cu's kernels do) and checked against the reference's own ggml-cpu ops, one-node graphs through
oracle/train_probe.cpp:
  OPT_STEP_ADAMW  bit for bit over a grid of lr, beta1, beta2, eps, wd (0 included) and iteration, with denormal and zero v;
  ARGMAX          ties (the last index wins), NaN at the start, middle and end of a row, runs of NaN, all-NaN and all -inf rows: the closed
                  form the device reduction computes equals ggml_vec_argmax_f32's sequential rule and ggml-cpu;
  REPEAT_BACK     the order of the adds over the repeats, bit for bit, on packed and strided (view) sources;
  OUT_PROD        the fused k-ascending chain bit for bit where ne0 is a multiple of 64 (ggml-cpu's SIMD body, AVX2 or AVX-512), within
                  NMSE 1e-12 otherwise; transposed src1 and broadcast batch dims;
  STEP            +-0, NaN, +-inf.
The EUNSUPPORTED / EINVAL codes of the eight checks (b200_op_checks.h), which the C ABI launchers and the plug-in's supports_op apply, are
pinned here too."""
import ctypes as C
import itertools

import numpy as np
import pytest

import ggml_b200 as g
from hostemu.emu import EINVAL, EUNSUPPORTED, I64, OK, desc, load, view_desc
from oracle import oracle as O
from oracle import train as TR
from oracle.pool import F32, I32, Source

OUT_PROD_NMSE = 1e-12


@pytest.fixture(scope="module")
def emu():
    L = load("train_emu")
    TD, vp = C.POINTER(g.TensorDesc), C.c_void_p
    L.emu_adamw.restype, L.emu_adamw.argtypes = None, [C.c_int64, vp, vp, vp, vp, vp]
    for fn in (L.emu_argmax_closed, L.emu_argmax_seq):
        fn.restype, fn.argtypes = C.c_int32, [vp, C.c_int64]
    L.emu_step.restype, L.emu_step.argtypes = None, [vp, vp, C.c_int64]
    for fn, n in ((L.emu_out_prod, 3), (L.emu_repeat_back, 2)):
        fn.restype, fn.argtypes = C.c_int, [TD] * n
    return L


@pytest.fixture(scope="module")
def checks():
    L = load("op_checks_emu")
    TD = C.POINTER(g.TensorDesc)
    for name, n in (("out_prod", 3), ("cross_entropy_loss", 3), ("cross_entropy_loss_back", 4), ("opt_step_adamw", 5), ("argmax", 2),
                    ("count_equal", 3), ("sum", 2), ("repeat_back", 2)):
        fn = getattr(L, "emu_check_" + name)
        fn.restype, fn.argtypes = C.c_int, [TD] * n
    return L


def u32(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


# ------------------------------------------------------------------ OPT_STEP_ADAMW
def adamw_params(lr, b1, b2, eps, wd, it):
    return np.array([lr, b1, b2, eps, wd, 1.0 / (1.0 - b1 ** it), 1.0 / (1.0 - b2 ** it)], dtype=np.float32)


def adamw_inputs(seed, n=257):
    rng = np.random.default_rng(seed)
    w = rng.standard_normal(n).astype(np.float32)
    gr = (rng.standard_normal(n) * 10.0 ** rng.integers(-6, 2, n)).astype(np.float32)
    m = (rng.standard_normal(n) * 0.1).astype(np.float32)
    v = np.abs(rng.standard_normal(n) * 10.0 ** rng.integers(-12, 0, n)).astype(np.float32)
    v[::7] = np.float32(1e-40)                           # denormal second moments
    v[3::11] = 0.0
    gr[5::13] = 0.0
    return w, gr, m, v


ADAMW_GRID = list(itertools.product([1e-3, 0.1], [0.9, 0.5], [0.999, 0.9], [1e-8, 1e-3], [0.0, 0.01], [1, 10]))


@pytest.mark.parametrize("lr,b1,b2,eps,wd,it", ADAMW_GRID)
def test_adamw_bit_identical(emu, lr, b1, b2, eps, wd, it):
    p = adamw_params(lr, b1, b2, eps, wd, it)
    w, gr, m, v = adamw_inputs(hash((lr, b1, b2, eps, wd, it)) % 1000)
    want_w, want_m, want_v = TR.opt_step_adamw("CPU", w, gr, m, v, p)
    hw, hm, hv = w.copy(), m.copy(), v.copy()
    emu.emu_adamw(w.size, hw.ctypes.data, gr.ctypes.data, hm.ctypes.data, hv.ctypes.data, p.ctypes.data)
    assert np.array_equal(u32(hm), u32(want_m)) and np.array_equal(u32(hv), u32(want_v))
    assert np.array_equal(u32(hw), u32(want_w))


# ------------------------------------------------------------------ ARGMAX
def argmax_rows():
    nan, inf = np.nan, np.inf
    rows = [
        [1, 3, 3, 2], [3, 3, 3], [-0.0, 0.0, -0.0], [0.0, -0.0],
        [nan, 1, 2, 0], [1, 5, nan, 2, 0], [1, 5, 2, nan], [1, 5, nan, nan], [nan, nan, nan], [nan],
        [-inf, -inf, -inf], [-inf], [2, nan, -inf, -inf], [4, nan, 1, nan, 0, 0, nan], [nan, 7, nan, nan, 3],
        [inf, 1, inf, nan, -inf], [5, 1, nan, 5, 5, nan],
    ]
    rng = np.random.default_rng(7)
    for n in (32, 100, 1000, 5438):
        x = rng.integers(-5, 5, n).astype(np.float32)          # many ties
        x[rng.integers(0, n, 3)] = np.nan
        rows.append(list(x))
    return [np.array(r, dtype=np.float32) for r in rows]


@pytest.mark.parametrize("i", range(len(argmax_rows())))
def test_argmax_rule(emu, i):
    x = argmax_rows()[i]
    want = int(TR.argmax("CPU", x.reshape(1, -1))[0])
    assert emu.emu_argmax_seq(x.ctypes.data, x.size) == want
    assert emu.emu_argmax_closed(x.ctypes.data, x.size) == want, list(x)


# ------------------------------------------------------------------ REPEAT_BACK
def repeat_back_cases():
    out = []
    for ne, nr, view in [((8, 6, 4, 2), (1, 1, 1, 1), False), ((8, 6, 4, 2), (2, 1, 1, 1), False), ((8, 6, 4, 2), (1, 2, 1, 1), False),
                         ((8, 6, 4, 2), (1, 1, 2, 1), False), ((8, 6, 4, 2), (1, 1, 1, 2), False), ((8, 6, 4, 2), (2, 2, 2, 2), False),
                         ((3, 5, 1, 1), (4, 3, 2, 5), False), ((1, 1, 1, 1), (7, 3, 2, 2), False),
                         ((8, 6, 4, 2), (2, 1, 1, 1), True), ((8, 6, 4, 2), (1, 2, 1, 1), True), ((8, 6, 4, 2), (1, 1, 2, 1), True),
                         ((8, 6, 4, 2), (1, 1, 1, 2), True)]:
        full = tuple(a * b for a, b in zip(ne, nr))
        if view:             # test-backend-ops' view: half of each repeated dim of a parent twice as large, the parent's strides
            parent = tuple(f * (2 if r > 1 else 1) for f, r in zip(full, nr))
            pnb = Source(F32, parent).nb
            src = Source(F32, full, parent_ne=parent, nb=pnb, seed=len(out))
        else:
            src = Source(F32, full, seed=len(out))
        out.append((src, ne))
    return out


def wide_parent(src: Source):
    rng = np.random.default_rng(500 + src.seed)           # wide exponents, so that the order of the adds shows in the bits
    x = (rng.standard_normal(src.parent_ne[::-1]) * 10.0 ** rng.integers(-4, 5, src.parent_ne[::-1])).astype(np.float32)
    return x


@pytest.mark.parametrize("i", range(len(repeat_back_cases())))
def test_repeat_back_order(emu, i):
    src, ne = repeat_back_cases()[i]
    parent = wide_parent(src)
    want = TR.repeat_back("CPU", src, ne, parent)
    got = np.zeros_like(want)
    rc = emu.emu_repeat_back(C.byref(view_desc(src, parent)), C.byref(desc(F32, ne, data=got.ctypes.data)))
    assert rc == OK
    assert np.array_equal(u32(got), u32(want))


# ------------------------------------------------------------------ OUT_PROD
def out_prod_cases():
    """(src0, src1) Sources: src0 [m, k, bs2, bs3] packed, src1 [n, k, bs2 nr2, bs3 nr3] packed or the transpose of a packed [k, n, ...]"""
    out = []
    for m, n, k, bs, nr, trans in [(64, 16, 16, (1, 1), (1, 1), False), (128, 32, 7, (3, 1), (2, 1), False), (256, 1, 1, (1, 3), (1, 2), False),
                                   (64, 10, 50, (1, 1), (1, 1), True), (192, 33, 129, (2, 2), (1, 2), True), (64, 5, 0, (1, 1), (1, 1), False),
                                   (100, 17, 23, (1, 1), (1, 1), False), (31, 9, 40, (2, 1), (1, 1), True), (784, 10, 64, (1, 1), (1, 1), True)]:
        a = Source(F32, (m, k, bs[0], bs[1]), seed=len(out))
        if trans:
            b = Source(F32, (k, n, bs[0] * nr[0], bs[1] * nr[1]), transpose=True, seed=100 + len(out))
        else:
            b = Source(F32, (n, k, bs[0] * nr[0], bs[1] * nr[1]), seed=100 + len(out))
        out.append((a, b))
    return out


def finite_parent(src: Source):
    rng = np.random.default_rng(900 + src.seed)
    return rng.uniform(-1, 1, src.parent_ne[::-1]).astype(np.float32)


@pytest.mark.parametrize("i", range(len(out_prod_cases())))
def test_out_prod_chain(emu, i):
    sa, sb = out_prod_cases()[i]
    pa, pb = finite_parent(sa), finite_parent(sb)
    want = TR.out_prod("CPU", sa, sb, pa, pb)
    got = np.zeros_like(want)
    ne_d = want.shape[::-1]
    rc = emu.emu_out_prod(C.byref(view_desc(sa, pa)), C.byref(view_desc(sb, pb)), C.byref(desc(F32, ne_d, data=got.ctypes.data)))
    assert rc == OK
    m = ne_d[0]
    body = m - m % 64
    assert np.array_equal(u32(got[..., :body]), u32(want[..., :body])), "the SIMD body's fused chain"
    if want.size and np.any(want):
        assert O.nmse(got.reshape(-1), want.reshape(-1)) <= OUT_PROD_NMSE
    # and against an f64 product
    a64 = pa.astype(np.float64)[..., : sa.ne[1], : sa.ne[0]]
    ne_b, _ = sb.view()
    b64 = np.swapaxes(pb.astype(np.float64), -1, -2) if sb.transpose else pb.astype(np.float64)
    a64 = np.repeat(np.repeat(a64, ne_b[2] // sa.ne[2], axis=1), ne_b[3] // sa.ne[3], axis=0)
    ref = np.einsum("...km,...kn->...nm", a64, b64)
    if ref.size and np.any(ref):
        assert O.nmse(got.reshape(-1), ref.reshape(-1)) <= OUT_PROD_NMSE


# ------------------------------------------------------------------ STEP
def test_step_specials(emu):
    x = np.array([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 1e-45, -1e-45, 3.0, -2.0], dtype=np.float32)
    want = TR.step("CPU", x)
    got = np.zeros_like(x)
    emu.emu_step(x.ctypes.data, got.ctypes.data, x.size)
    assert np.array_equal(u32(got), u32(want))
    assert list(got) == [0, 0, 0, 0, 1, 0, 1, 0, 1, 0]


# ------------------------------------------------------------------ the checks' codes
def test_check_codes(checks):
    b = C.byref
    # OUT_PROD
    a, y, d = desc(F32, (8, 4, 2, 1)), desc(F32, (5, 4, 4, 1)), desc(F32, (8, 5, 4, 1))
    assert checks.emu_check_out_prod(b(a), b(y), b(d)) == OK
    assert checks.emu_check_out_prod(b(a), b(desc(F32, (5, 4, 4, 1), nb=(16, 4, 80, 320))), b(d)) == OK       # transposed src1
    assert checks.emu_check_out_prod(b(desc(1, (8, 4, 2, 1))), b(y), b(d)) == EUNSUPPORTED                    # f16 src0
    assert checks.emu_check_out_prod(b(desc(F32, (8, 4, 2, 1), nb=(16, 4, 128, 256))), b(y), b(d)) == EUNSUPPORTED
    assert checks.emu_check_out_prod(b(a), b(y), b(desc(F32, (8, 5, 4, 1), nb=(4, 64, 320, 1280)))) == EUNSUPPORTED
    assert checks.emu_check_out_prod(b(a), b(desc(F32, (5, 3, 4, 1))), b(d)) == EINVAL                        # K differs
    assert checks.emu_check_out_prod(b(desc(F32, (8, 4, 3, 1))), b(y), b(d)) == EINVAL                        # 4 % 3
    # CROSS_ENTROPY_LOSS / _BACK
    x, s = desc(F32, (10, 5)), desc(F32, (1,))
    assert checks.emu_check_cross_entropy_loss(b(x), b(x), b(s)) == OK
    assert checks.emu_check_cross_entropy_loss(b(x), b(desc(F32, (10, 4))), b(s)) == EINVAL
    assert checks.emu_check_cross_entropy_loss(b(x), b(x), b(desc(F32, (2,)))) == EINVAL
    assert checks.emu_check_cross_entropy_loss(b(desc(F32, (10, 5), nb=(20, 4, 200, 200))), b(x), b(s)) == EUNSUPPORTED
    assert checks.emu_check_cross_entropy_loss(b(desc(1, (10, 5))), b(x), b(s)) == EUNSUPPORTED
    assert checks.emu_check_cross_entropy_loss_back(b(s), b(x), b(x), b(x)) == OK
    assert checks.emu_check_cross_entropy_loss_back(b(desc(F32, (2,))), b(x), b(x), b(x)) == EINVAL
    assert checks.emu_check_cross_entropy_loss_back(b(s), b(x), b(x), b(desc(F32, (10, 5), nb=(4, 48, 240, 240)))) == EUNSUPPORTED
    # OPT_STEP_ADAMW
    w, p = desc(F32, (10, 5, 4, 3)), desc(F32, (7,))
    assert checks.emu_check_opt_step_adamw(b(w), b(w), b(w), b(w), b(p)) == OK
    assert checks.emu_check_opt_step_adamw(b(w), b(w), b(w), b(w), b(desc(F32, (6,)))) == EINVAL
    assert checks.emu_check_opt_step_adamw(b(w), b(desc(F32, (10, 5, 4, 2))), b(w), b(w), b(p)) == EINVAL
    assert checks.emu_check_opt_step_adamw(b(w), b(w), b(desc(F32, (10, 5, 4, 3), nb=(4, 48, 240, 960))), b(w), b(p)) == EUNSUPPORTED
    assert checks.emu_check_opt_step_adamw(b(desc(1, (10, 5, 4, 3))), b(w), b(w), b(w), b(p)) == EUNSUPPORTED
    # ARGMAX
    assert checks.emu_check_argmax(b(desc(F32, (100, 10))), b(desc(I32, (10,)))) == OK
    assert checks.emu_check_argmax(b(desc(F32, (100, 10))), b(desc(F32, (10,)))) == EUNSUPPORTED
    assert checks.emu_check_argmax(b(desc(F32, (100, 10), nb=(40, 4, 400, 400))), b(desc(I32, (10,)))) == EUNSUPPORTED
    assert checks.emu_check_argmax(b(desc(F32, (100, 10, 2))), b(desc(I32, (10,)))) == EINVAL
    assert checks.emu_check_argmax(b(desc(F32, (100, 10))), b(desc(I32, (9,)))) == EINVAL
    assert checks.emu_check_argmax(b(desc(F32, (0, 10))), b(desc(I32, (10,)))) == EINVAL
    # COUNT_EQUAL
    ci, c64 = desc(I32, (4, 500)), desc(I64, (1,))
    assert checks.emu_check_count_equal(b(ci), b(ci), b(c64)) == OK
    assert checks.emu_check_count_equal(b(ci), b(desc(I32, (4, 499))), b(c64)) == EINVAL
    assert checks.emu_check_count_equal(b(ci), b(ci), b(desc(I32, (1,)))) == EUNSUPPORTED
    assert checks.emu_check_count_equal(b(desc(I32, (4, 5, 3))), b(desc(I32, (4, 5, 3))), b(c64)) == EUNSUPPORTED
    # SUM
    assert checks.emu_check_sum(b(desc(F32, (10, 5, 4, 3))), b(s)) == OK
    assert checks.emu_check_sum(b(desc(F32, (10, 5), nb=(20, 4, 200, 200))), b(s)) == EUNSUPPORTED
    assert checks.emu_check_sum(b(desc(F32, (10, 5))), b(desc(F32, (2,)))) == EINVAL
    # REPEAT_BACK
    assert checks.emu_check_repeat_back(b(desc(F32, (16, 6, 4, 2))), b(desc(F32, (8, 6, 4, 2)))) == OK
    assert checks.emu_check_repeat_back(b(desc(I32, (16, 6, 4, 2))), b(desc(I32, (8, 6, 4, 2)))) == EUNSUPPORTED
    assert checks.emu_check_repeat_back(b(desc(F32, (16, 6), nb=(8, 128, 768, 768))), b(desc(F32, (8, 6)))) == EUNSUPPORTED
    assert checks.emu_check_repeat_back(b(desc(F32, (15, 6))), b(desc(F32, (8, 6)))) == EINVAL
