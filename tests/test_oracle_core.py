"""CPU-only: the f64 references of oracle/core.py against ggml-cpu (oracle/_ref/libggml_core_probe.so), so that a wrong reference cannot
pass a wrong device kernel in tests/test_gpu_core_ops.py.
  - bit-exact: GET_ROWS of f32, f16 and all 21 block formats (Oracle.dequantize); ADD / SUB / MUL / DIV with broadcast, views and in
    place, +-0, +-inf, NaN and subnormal operands; SCALE; DIAG_MASK_INF; SQR, SQRT, NEG, ABS, RELU, STEP; the float CPY / CONT / DUP
    (round to nearest even, 65520 -> inf, NaN compared by isnan);
  - GELU and GELU_QUICK on every f16 bit pattern (and +-10, +-65519, +-65520): the reference reproduces ggml-cpu's f16 tables exactly;
  - within a few ulp of f64: TANH, EXP, SIGMOID, SILU (ggml-cpu's vector ggml_v_silu), SIN and COS;
  - NORM and RMS_NORM to f32 round-off of the reference that rounds the mean to f32 as ggml-cpu does."""
import numpy as np
import pytest

from oracle import core as K
from oracle import oracle as O
from oracle.pool import F32, Source

# ggml-cpu against the f64 reference, in ulp (measured on x86-64: TANH 1.97, SIGMOID 1.83, EXP 0.50, SIN 0.54, COS 0.55, SILU 3.15)
CPU_ULP = {K.TANH: 3.0, K.EXP: 1.0, K.SIGMOID: 3.0, K.SILU: 6.0, K.SIN: 1.0, K.COS: 1.0}
NORM_NMSE = 6e-14                 # f32 round-off of (x - mean), the scale and the product: 6.4e-15 measured


@pytest.fixture(scope="module", autouse=True)
def need_probe():
    if not (O.REF_DIR / "libggml_core_probe.so").exists():
        pytest.skip("libggml_core_probe.so not built (oracle/_ref needs the reference tree)")


@pytest.mark.parametrize("case", K.get_rows_grid(), ids=lambda c: f"{O.TYPE_NAMES[c[0].type]}-{c[0].ne}-{c[2]}")
def test_get_rows_is_the_oracle_dequantization(case):
    src, n, order = case
    parent = K.get_rows_parent(src)
    ids = K.get_rows_ids(n, src.ne[2], src.ne[3], src.ne[1], order, src.seed)
    got = K.get_rows("CPU", src, parent, ids)
    assert K.same_bits(got, K.get_rows_reference(src, parent, ids)).all()


@pytest.mark.parametrize("case", [c for c in K.binary_grid() if c[4]], ids=lambda c: f"{K.BIN_NAMES[c[0]]}-{c[1].ne}-{c[2].ne}{'-inplace' * c[3]}")
def test_binary_ops_are_correctly_rounded(case):
    op, s0, s1, inplace, _ = case
    p0, p1 = K.binary_values(s0), K.binary_values(s1)
    want = K.binary_reference(op, K.logical(s0, p0), K.logical(s1, p1))
    got = K.binary("CPU", op, s0, p0, s1, p1, inplace)
    if inplace:
        p = p0.copy()
        ne, nb = s0.view()
        np.lib.stride_tricks.as_strided(p.reshape(-1)[s0.offs // 4:], shape=ne[::-1], strides=nb[::-1])[...] = want
        want = p
    assert K.same_bits(got, want).all()


def test_binary_edge_operands_are_present():
    """DIV meets +-0 and subnormal divisors and 0 / 0 in the grid; the reference's results include +-inf and NaN"""
    s = Source(F32, (40, 5, 3, 2))
    x = K.binary_values(s)
    r = K.binary_reference(K.DIV, x, x[:, :, :1, :])
    assert np.isnan(r).any() and np.isposinf(r).any() and np.isneginf(r).any()
    assert (np.abs(x[(x != 0) & np.isfinite(x)]) < K.FLT_MIN).any()


@pytest.mark.parametrize("op", range(14), ids=lambda o: K.UNARY_NAMES[o])
def test_unary_reference_matches_ggml_cpu(op):
    if op in K.TABLE_UNARY:
        x = K.f16_inputs()
    else:
        x = K.unary_values(op)
    got, ref = K.unary("CPU", op, x), K.unary_reference(op, x)
    if op in K.EXACT_UNARY or op in K.TABLE_UNARY:
        bad = ~K.same_bits(got, ref)
        assert not bad.any(), (K.UNARY_NAMES[op], x[bad][:8], got[bad][:8], ref[bad][:8])
    else:
        e = K.ulp_error(got, ref, K.SILU_TINY if op == K.SILU else K.FLT_MIN)
        assert e.max() <= CPU_ULP[op], (K.UNARY_NAMES[op], float(e.max()), float(x[np.argmax(e)]))


def test_gelu_quick_table_is_not_the_f32_formula():
    """the f32 formula x / (1 + expf(-1.702 x)) without the f16 roundings differs from ggml-cpu on most f16 inputs: the bit-exact check
    above tells the two apart"""
    x = K.f16_inputs()
    fin = np.isfinite(x) & (np.abs(x) < 65504)
    f = np.float32
    with np.errstate(all="ignore"):
        plain = x * (f(1.0) / (f(1.0) + K._expf(f(-1.702) * x)))
    assert (~K.same_bits(plain, K.unary("CPU", K.GELU_QUICK, x)))[fin].sum() > fin.sum() // 2
    edges = K.gelu_quick_table(np.array([65519.0, 65520.0, -65519.0, -65520.0], np.float32))
    assert edges[0] == 65504.0 and np.isposinf(edges[1]) and edges[2] == 0.0 and np.isnan(edges[3])


@pytest.mark.parametrize("case", K.norm_grid(), ids=lambda c: f"{'rms' if c[0] else 'norm'}-{c[2].ne}-eps{c[1]:g}-off{c[3]:g}{'-zeros' * c[4]}")
def test_norm_reference_matches_ggml_cpu(case):
    rms, eps, src, offset, zero_rows = case
    parent = K.norm_values(src.parent_ne, offset, src.seed, zero_rows)
    got = K.norm("CPU", rms, eps, src, parent)
    ref = K.norm_reference(K.logical(src, parent), eps, rms)
    nan = np.isnan(ref)                       # eps 0 over a zero row (or NORM of one element): 0 * (1 / sqrtf(0)) on both backends
    assert (np.isnan(got) == nan).all() and nan.any() == (eps == 0.0 and (zero_rows or (src.ne[0] == 1 and not rms)))
    assert K.nmse64(got[~nan], ref[~nan]) <= NORM_NMSE, K.nmse64(got[~nan], ref[~nan])


def test_scale_and_diag_mask_inf_are_exact():
    x = np.random.default_rng(5).standard_normal((2, 3, 7, 19)).astype(np.float32)
    for scale, n_past in ((0.125, 0), (-3.7, 4), (1e-30, 30)):
        s, m = K.scale_mask("CPU", x, scale, n_past)
        want_s = (x.astype(np.float64) * np.float32(scale)).astype(np.float32)
        i1, i0 = np.arange(7)[:, None], np.arange(19)[None, :]
        assert K.same_bits(s, want_s).all() and K.same_bits(m, np.where(i0 > n_past + i1, -np.inf, want_s)).all()


@pytest.mark.parametrize("case", K.cpy_grid(), ids=lambda c: f"{('cpy', 'cont', 'dup')[c[0]]}-{c[1].type}-{c[1].ne}{'T' * c[1].transpose}")
def test_float_cpy_rounds_to_nearest_even(case):
    op, src, dst = case
    parent = K.cpy_values(src)
    if op == 0:
        dst_in = K.cpy_dst_in(dst)
        got, want = K.cpy("CPU", 0, src, parent, dst, dst_in), K.cpy_expected(src, parent, dst, dst_in)
    else:
        got, want = K.cpy("CPU", op, src, parent), K.cpy_reference(K.logical(src, parent), src.type)
    assert K.same_bits(got, want).all()


def test_cpy_values_hold_the_f16_edges():
    y = K.cpy_reference(K.cpy_values(Source(F32, (37, 5, 3, 1))), 1).astype(np.float32)
    assert np.isposinf(y).any() and (y == 65504.0).any() and (np.abs(y[(y != 0) & np.isfinite(y)]) < 6.1e-5).any() and np.isnan(y).any()
