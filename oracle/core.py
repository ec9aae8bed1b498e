"""TEST INFRASTRUCTURE ONLY: the small ops either side of every mat-mul -- GET_ROWS, ADD / SUB / MUL / DIV with broadcast, NORM / RMS_NORM,
SCALE, DIAG_MASK_INF, the unary functions, SQR / SQRT / SIN / COS and the float CPY / CONT / DUP -- as cases, their f64 references, and the
reference's ops through oracle/_ref/libggml_core_probe.so (oracle/core_probe.cpp), which also runs the two chains the plug-in fuses
(NORM -> MUL -> ADD and SCALE -> DIAG_MASK_INF -> SOFT_MAX).

Every node input is a `pool.Source` (a view of a parent); `logical` reads the values a view sees.  The references compute in f64 and round
once to f32 where ggml-cpu's op is one IEEE operation (so they are bit-exact there), follow ggml-cpu's f32 roundings where it has them (the
norms' mean and scale) and emulate ggml-cpu's f16 tables for GELU and GELU_QUICK.  `get_rows(dev, ...)` etc. evaluate on a named ggml
device ("CPU": ggml-cpu; "B2000": the plug-in, once loaded with oracle.Ref().load_backend)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import oracle as O
from .pool import ES, F16, F32, I32, Source
from .probe import probe_lib, result

ADD, MUL, SUB, DIV = 0, 1, 2, 3                 # the kernel library's (and probe_binary's) op codes
BIN_NAMES = {ADD: "add", MUL: "mul", SUB: "sub", DIV: "div"}
# GGML_B200_UNARY_* (include/ggml-b200.h), the codes probe_unary and ggml_b200_op_unary take
GELU, SILU, RELU, TANH, NEG, ABS, GELU_QUICK, SIGMOID, EXP, SQR, SQRT, SIN, COS, STEP = range(14)
UNARY_NAMES = ["gelu", "silu", "relu", "tanh", "neg", "abs", "gelu_quick", "sigmoid", "exp", "sqr", "sqrt", "sin", "cos", "step"]
EXACT_UNARY = (RELU, NEG, ABS, SQR, SQRT, STEP)  # one IEEE operation (or none): bit-exact on every backend
TABLE_UNARY = (GELU, GELU_QUICK)                 # ggml-cpu reads an f16 -> f16 table
FLT_MIN = float(np.finfo(np.float32).tiny)
BLOCK_TYPES = (O.Q4_0, O.Q4_1, O.Q5_0, O.Q5_1, O.Q8_0, O.IQ4_NL, O.Q2_K, O.Q3_K, O.Q4_K, O.Q5_K, O.Q6_K, O.IQ4_XS, O.IQ2_XXS, O.IQ2_XS,
               O.IQ2_S, O.IQ3_XXS, O.IQ3_S, O.IQ1_S, O.IQ1_M, O.TQ1_0, O.TQ2_0)
_orc = None


def orc() -> O.Oracle:
    global _orc
    if _orc is None:
        _orc = O.Oracle()
    return _orc


def row_bytes(t, n):
    return n * ES[t] if t in ES else orc().row_size(t, n)


def block_source(t, ne, parent_ne=None, seed=0) -> Source:
    """a Source of type t (block formats too: nb from the row size) over a packed parent"""
    pne = tuple(parent_ne or ne) + (1,) * (4 - len(parent_ne or ne))
    rb = row_bytes(t, pne[0])
    return Source(t, ne, parent_ne=pne, nb=(rb, rb * pne[1], rb * pne[1] * pne[2]), seed=seed)


def logical(src: Source, parent: np.ndarray) -> np.ndarray:
    """the elements a float (or i32) view reads from its parent, numpy order of its logical ne (transposition applied)"""
    ne, nb = src.view()
    flat = np.ascontiguousarray(parent).reshape(-1)
    st = np.lib.stride_tricks.as_strided(flat[src.offs // ES[src.type]:], shape=ne[::-1], strides=nb[::-1])
    return np.ascontiguousarray(st)


def f16(x) -> np.ndarray:
    """f32 -> f16 -> f32, rounding to nearest even (numpy's conversion): 65520 and above overflow to inf, 65519 rounds to 65504"""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(x, dtype=np.float32).astype(np.float16).astype(np.float32)


def nmse64(got, ref) -> float:
    """sum (got - ref)^2 / sum ref^2 in f64 (ref: the f64 reference)"""
    g, r = np.asarray(got, np.float64).ravel(), np.asarray(ref, np.float64).ravel()
    den = float(np.sum(r * r))
    return float(np.sum((g - r) ** 2)) / den if den > 0 else float(np.sum((g - r) ** 2))


def same_bits(a, b) -> np.ndarray:
    """element-wise: identical f32 / f16 bits, or both NaN (a NaN's payload is not part of any op's result)"""
    a, b = np.asarray(a), np.asarray(b)
    u = np.uint32 if a.dtype == np.float32 else np.uint16
    return (a.view(u) == b.view(u)) | (np.isnan(a) & np.isnan(b))


# ------------------------------------------------------------------ GET_ROWS
def get_rows_parent(src: Source) -> np.ndarray:
    """the parent's bytes (uint8): random valid blocks; f16 / f32 normals with +-inf, -0 and subnormals among them (f32: NaN too)"""
    rng = np.random.default_rng(20000 + src.seed)
    n = int(np.prod(src.parent_ne))
    if src.type in (F32, F16):
        x = rng.standard_normal(n).astype(np.float32)
        x[3::41], x[5::43], x[7::47] = np.inf, -np.inf, -0.0
        x[11::53] = 3e-6 if src.type == F16 else 1e-40
        if src.type == F32:
            x[13::59] = np.nan
        return x.astype(np.float16 if src.type == F16 else np.float32).view(np.uint8)
    return O.random_blocks(src.type, n // orc().blck_size(src.type), rng)


def get_rows_ids(n, ne11, ne12, rows, order="random", seed=0) -> np.ndarray:
    """i32 [ne12, ne11, n]: random (with repeats), descending or repeated row ids below `rows`"""
    rng = np.random.default_rng(21000 + seed)
    if order == "descending":
        ids = np.broadcast_to((rows - 1 - np.arange(n) % rows), (ne12, ne11, n))
    elif order == "repeated":
        ids = np.full((ne12, ne11, n), rows // 2)
        ids[..., ::3] = rows - 1
    else:
        ids = rng.integers(0, rows, (ne12, ne11, n))
    return np.ascontiguousarray(ids, dtype=np.int32)


def get_rows_reference(src: Source, parent: np.ndarray, ids: np.ndarray) -> np.ndarray:
    """f32 [ne12, ne11, n, ne0]: row ids[i12, i11, i10] of src's matrix (i11, i12), decoded (Oracle.dequantize for the block formats)"""
    ne0 = src.ne[0]
    rb = row_bytes(src.type, ne0)
    nb1, nb2, nb3 = src.nb
    out = np.empty(ids.shape + (ne0,), np.float32)
    for i12 in range(ids.shape[0]):
        for i11 in range(ids.shape[1]):
            for i10, r in enumerate(ids[i12, i11]):
                o = src.offs + int(r) * nb1 + i11 * nb2 + i12 * nb3
                raw = parent[o: o + rb]
                if src.type == F32:
                    out[i12, i11, i10] = raw.view(np.float32)
                elif src.type == F16:
                    out[i12, i11, i10] = raw.view(np.float16).astype(np.float32)
                else:
                    out[i12, i11, i10] = orc().dequantize(src.type, raw, ne0)
    return out


# ------------------------------------------------------------------ ADD / SUB / MUL / DIV
def binary_values(src: Source) -> np.ndarray:
    """an f32 parent of normals with 0, -0, +-inf, NaN and subnormals among them (divisors of +-0 and subnormals: DIV's edge cases)"""
    rng = np.random.default_rng(22000 + src.seed)
    x = rng.standard_normal(src.parent_ne[::-1]).astype(np.float32)
    f = x.reshape(-1)
    f[2::17], f[4::19], f[6::23], f[8::29] = 0.0, -0.0, 1e-40, -3e-39
    f[10::31], f[12::37], f[14::41] = np.inf, -np.inf, np.nan
    return x


def binary_reference(op, a, b) -> np.ndarray:
    """a (op) b with b tiled over a (ggml's whole-repeat broadcast), in f64 and rounded once to f32: the correctly rounded f32 result"""
    reps = [sa // sb for sa, sb in zip(a.shape, b.shape)]
    x, y = a.astype(np.float64), np.tile(b, reps).astype(np.float64)
    with np.errstate(all="ignore"):
        r = x + y if op == ADD else x * y if op == MUL else x - y if op == SUB else x / y
        return r.astype(np.float32)


# ------------------------------------------------------------------ NORM / RMS_NORM
def norm_reference(x, eps: float, rms: bool, f32_mean: bool = True) -> np.ndarray:
    """f64 NORM / RMS_NORM along the last axis.  f32_mean: as ggml-cpu writes it, the mean (NORM) rounded to f32 before the subtraction;
    otherwise the exact one"""
    x = np.asarray(x, np.float64)
    n = x.shape[-1]
    with np.errstate(all="ignore"):
        if rms:
            v = x
            var = np.sum(x * x, axis=-1, keepdims=True) / n
        else:
            mean = np.sum(x, axis=-1, keepdims=True) / n
            if f32_mean:
                mean = mean.astype(np.float32).astype(np.float64)
            v = x - mean
            var = np.sum(v * v, axis=-1, keepdims=True) / n
        return v / np.sqrt(var + np.float64(np.float32(eps)))


def norm_values(ne, offset: float, seed: int, zero_rows: bool = False) -> np.ndarray:
    """f32 [ne3, ne2, ne1, ne0] normals plus a common offset; zero_rows: every third row all zeros"""
    rng = np.random.default_rng(23000 + seed)
    x = (rng.standard_normal(ne[::-1]) + offset).astype(np.float32)
    if zero_rows:
        x.reshape(-1, ne[0])[::3] = 0.0
    return x


# ------------------------------------------------------------------ unary
def _expf(x):
    """expf, correctly rounded (glibc's is within 0.502 ulp; its rare misroundings are what a pinned exception list covers)"""
    with np.errstate(all="ignore"):
        return np.exp(x.astype(np.float64)).astype(np.float32)


def _tanhf(x):
    return np.tanh(x.astype(np.float64)).astype(np.float32)


def gelu_table(x) -> np.ndarray:
    """ggml-cpu's GELU (ggml_vec_gelu_f32 with GGML_GELU_FP16): x <= -10: 0; x >= 10: x; otherwise x rounded to f16, 0.5 x (1 + tanhf(
    sqrt(2/pi) x (1 + 0.044715 x x))) in f32 without contraction, rounded to f16"""
    x = np.asarray(x, np.float32)
    h = f16(x)
    f = np.float32
    with np.errstate(all="ignore"):
        inner = f(0.79788456080286535587989211986876) * h * (f(1.0) + f(0.044715) * h * h)
        g = f16(f(0.5) * h * (f(1.0) + _tanhf(inner)))
    return np.where(x <= -10.0, f(0.0), np.where(x >= 10.0, x, g)).astype(np.float32)


def gelu_quick_table(x) -> np.ndarray:
    """ggml-cpu's GELU_QUICK (GGML_GELU_QUICK_FP16): x rounded to f16, x (1 / (1 + expf(-1.702 x))) in f32, rounded to f16.  No cut-offs:
    |x| >= 65520 reads the table at +-inf, which holds +inf and NaN (-inf * 0)"""
    h = f16(x)
    f = np.float32
    with np.errstate(all="ignore"):
        return f16(h * (f(1.0) / (f(1.0) + _expf(f(-1.702) * h))))


def unary_reference(op: int, x) -> np.ndarray:
    """f64 (f32 for the two table functions, whose table is the definition) value of `op` at x; the exact ops rounded once to f32 are
    bit-exact"""
    if op == GELU:
        return gelu_table(x)
    if op == GELU_QUICK:
        return gelu_quick_table(x)
    v = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        r = {SILU: lambda: v / (1.0 + np.exp(-v)), RELU: lambda: np.where(v > 0, v, 0.0), TANH: lambda: np.tanh(v), NEG: lambda: -v,
             ABS: lambda: np.abs(v), SIGMOID: lambda: 1.0 / (1.0 + np.exp(-v)), EXP: lambda: np.exp(v), SQR: lambda: v * v,
             SQRT: lambda: np.sqrt(v), SIN: lambda: np.sin(v), COS: lambda: np.cos(v), STEP: lambda: np.where(v > 0, 1.0, 0.0)}[op]()
        return r if op not in EXACT_UNARY else r.astype(np.float32)


def unary_values(op: int, n: int = 4096, seed: int = 0) -> np.ndarray:
    """f32 inputs for `op`: its working range (SIN / COS up to |x| = 1e4, EXP / SILU / SIGMOID past the f32 overflow of exp), then +-0,
    +-inf, NaN, subnormals, FLT_MIN, FLT_MAX and the f16 edges 65504 / 65519 / 65520"""
    rng = np.random.default_rng(24000 + 31 * op + seed)
    span = {SIN: 1e4, COS: 1e4, EXP: 100.0, SILU: 110.0, SIGMOID: 110.0, TANH: 12.0, SQRT: 1e3, SQR: 1e4}.get(op, 12.0)
    x = np.concatenate([rng.uniform(-span, span, n // 2), rng.standard_normal(n // 4),
                        rng.uniform(-1, 1, n // 4) * 10.0 ** rng.integers(-30, 30, n // 4)])
    edges = [0.0, -0.0, np.inf, -np.inf, np.nan, 1e-40, -1e-40, 1.4e-45, -1.4e-45, FLT_MIN, -FLT_MIN, 3.4e38, -3.4e38, 65504.0, -65504.0,
             65519.0, -65519.0, 65520.0, -65520.0, 10.0, -10.0, 88.72, -88.72, 89.0, -89.0, 103.9, -103.9, 104.0, -104.0, 1e30, -1e30]
    return np.concatenate([x, edges]).astype(np.float32)


def f16_inputs() -> np.ndarray:
    """every f16 bit pattern as an f32 input (NaNs included), then +-10, +-65519 and +-65520"""
    return np.concatenate([np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16).astype(np.float32),
                           np.array([10.0, -10.0, 65519.0, -65519.0, 65520.0, -65520.0], np.float32)])


SILU_TINY = 1e-36       # SILU's results below this are compared absolutely: x / (1 + expf(-x)) is -0 where expf(-x) overflows (x below
                        # -88.72 on the device, -88.38 in ggml-cpu's vector expf), where the true value is at most 88.72 e^-88.72 = 2.9e-37


def ulp_error(got, ref, tiny: float = FLT_MIN) -> np.ndarray:
    """|got - ref| in units of the f32 spacing at ref (ref f64); where |ref| < tiny the absolute difference in units of tiny.  inf where
    the special values disagree (an infinite or NaN result on one side only, or infinities of different signs)"""
    g, r = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    with np.errstate(all="ignore"):
        r32 = r.astype(np.float32)
        sp = np.spacing(np.abs(r32).astype(np.float32)).astype(np.float64)
        e = np.where(np.abs(r) < tiny, np.abs(g - r) / tiny, np.abs(g - r) / sp)
    special = ~np.isfinite(r32) | ~np.isfinite(g)
    agree = (np.isnan(r32) & np.isnan(g)) | (np.isinf(r32) & (g == r32))
    return np.where(special, np.where(agree, 0.0, np.inf), e)


# ------------------------------------------------------------------ float CPY / CONT / DUP
def cpy_values(src: Source) -> np.ndarray:
    """the parent's elements: f32 normals with the f16 edges among them (65504, 65519 -> 65504, 65520 -> inf, 1e5, f16 subnormals,
    values that underflow f16), +-inf, NaN and -0; f16 the same values rounded"""
    rng = np.random.default_rng(25000 + src.seed)
    x = (rng.standard_normal(src.parent_ne[::-1]) * 4.0).astype(np.float32)
    f = x.reshape(-1)
    for k, v in enumerate([65504.0, 65519.0, 65520.0, -65520.0, 1e5, 3e-5, -2e-7, 5.9e-8, 2.9e-8, 1e-9, np.inf, -np.inf, np.nan, -0.0,
                           65519.99, -65505.0]):
        f[k::29] = v
    return x if src.type == F32 else f16(x).astype(np.float16)


def cpy_reference(src_vals: np.ndarray, dst_type: int) -> np.ndarray:
    """the values a float copy writes: conversions round to nearest even (f16 -> f32 and f16 -> f16 exact)"""
    with np.errstate(over="ignore"):
        return src_vals.astype(np.float32) if dst_type == F32 else src_vals.astype(np.float16)


def cpy_dst_in(dst: Source) -> np.ndarray:
    """the destination parent before the copy: a recognisable fill (every element -7.25), so untouched bytes are checked"""
    return np.full(dst.parent_ne[::-1], -7.25, dtype=np.float32 if dst.type == F32 else np.float16)


def cpy_expected(src: Source, src_parent, dst: Source, dst_in) -> np.ndarray:
    """the destination parent after ggml_cpy(src view, dst view)"""
    vals = cpy_reference(logical(src, src_parent), dst.type).reshape(-1)
    out = dst_in.copy()
    ne, nb = dst.view()
    es = ES[dst.type]
    v = np.lib.stride_tricks.as_strided(out.reshape(-1)[dst.offs // es:], shape=ne[::-1], strides=nb[::-1])
    v[...] = vals.reshape(ne[::-1])
    return out


# ------------------------------------------------------------------ the probe
SIGNATURES = {
    "probe_get_rows": [C.c_char_p] + [C.c_void_p] * 5,
    "probe_binary": [C.c_char_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p],
    "probe_norm": [C.c_char_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p],
    "probe_unary": [C.c_char_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p],
    "probe_scale_mask": [C.c_char_p, C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p],
    "probe_cpy": [C.c_char_p, C.c_int] + [C.c_void_p] * 5,
    "probe_norm_affine": [C.c_char_p, C.c_int, C.c_float] + [C.c_void_p] * 7,
    "probe_scale_mask_softmax": [C.c_char_p, C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_void_p],
}


def _lib():
    return probe_lib("core", "make -C oracle -f core.mk core", SIGNATURES)


def _ne(shape) -> np.ndarray:
    """ggml ne[4] of a numpy shape"""
    return np.array(list(shape[::-1]) + [1] * (4 - len(shape)), dtype=np.int64)


def get_rows(dev: str, src: Source, parent: np.ndarray, ids: np.ndarray, raw: bool = False):
    """GET_ROWS on `dev`: f32 [ne12, ne11, n, ne0]"""
    ids = np.ascontiguousarray(ids, np.int32)
    ss, si = src.spec(), Source(I32, _ne(ids.shape)).spec()          # held: read through raw pointers
    out = np.zeros(ids.shape + (src.ne[0],), np.float32)
    rc = _lib().probe_get_rows(dev.encode(), ss.ctypes.data, si.ctypes.data, parent.ctypes.data, ids.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_get_rows({dev}, {O.TYPE_NAMES[src.type]} {src.ne})", out)


def binary(dev: str, op: int, s0: Source, p0: np.ndarray, s1: Source, p1: np.ndarray, inplace: bool = False, raw: bool = False):
    """ADD / MUL / SUB / DIV on `dev`: not in place the packed result (numpy order of s0's logical ne); in place s0's whole parent"""
    out = np.zeros(p0.shape if inplace else s0.view()[0][::-1], np.float32)
    sp0, sp1 = s0.spec(), s1.spec()
    rc = _lib().probe_binary(dev.encode(), op, sp0.ctypes.data, sp1.ctypes.data, int(inplace), p0.ctypes.data, p1.ctypes.data,
                             out.ctypes.data)
    return result(rc, raw, f"probe_binary({dev}, {BIN_NAMES[op]}, {s0.ne}, {s1.ne})", out)


def norm(dev: str, rms: bool, eps: float, src: Source, parent: np.ndarray, raw: bool = False):
    out, sp = np.zeros(src.ne[::-1], np.float32), src.spec()
    rc = _lib().probe_norm(dev.encode(), int(rms), eps, sp.ctypes.data, parent.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_norm({dev}, rms={rms}, {src.ne})", out)


def unary(dev: str, op: int, x: np.ndarray, raw: bool = False):
    """a unary function of a packed f32 x on `dev`"""
    x = np.ascontiguousarray(x, np.float32)
    out, sp = np.zeros_like(x), Source(F32, _ne(x.shape)).spec()
    rc = _lib().probe_unary(dev.encode(), op, sp.ctypes.data, x.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_unary({dev}, {UNARY_NAMES[op]})", out)


def scale_mask(dev: str, x: np.ndarray, scale: float, n_past: int, raw: bool = False):
    """(SCALE, DIAG_MASK_INF) of the two-node graph on `dev`"""
    x = np.ascontiguousarray(x, np.float32)
    s, m, ne = np.zeros_like(x), np.zeros_like(x), _ne(x.shape)
    rc = _lib().probe_scale_mask(dev.encode(), ne.ctypes.data, scale, n_past, x.ctypes.data, s.ctypes.data, m.ctypes.data)
    return result(rc, raw, f"probe_scale_mask({dev}, {x.shape})", (s, m))


def cpy(dev: str, op: int, src: Source, parent: np.ndarray, dst: Source | None = None, dst_in: np.ndarray | None = None, raw: bool = False):
    """op 0: ggml_cpy into dst's view, the whole destination parent afterwards; 1 / 2: ggml_cont / ggml_dup, the packed result"""
    out = np.zeros_like(dst_in) if op == 0 else np.zeros(src.view()[0][::-1], parent.dtype)
    ss, sd = src.spec(), None if dst is None else dst.spec()
    rc = _lib().probe_cpy(dev.encode(), op, ss.ctypes.data, None if sd is None else sd.ctypes.data, parent.ctypes.data,
                          None if dst_in is None else dst_in.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_cpy({dev}, {('cpy', 'cont', 'dup')[op]}, {src.ne})", out)


def norm_affine(dev: str, rms: bool, eps: float, x: np.ndarray, gain: np.ndarray, bias: np.ndarray, raw: bool = False):
    """(NORM, MUL(gain), ADD(bias)) of the three-node graph on `dev`"""
    x = np.ascontiguousarray(x, np.float32)
    outs, ne = [np.zeros_like(x) for _ in range(3)], _ne(x.shape)
    rc = _lib().probe_norm_affine(dev.encode(), int(rms), eps, ne.ctypes.data, x.ctypes.data, gain.ctypes.data, bias.ctypes.data,
                                  *(o.ctypes.data for o in outs))
    return result(rc, raw, f"probe_norm_affine({dev}, rms={rms}, {x.shape})", tuple(outs))


def scale_mask_softmax(dev: str, x: np.ndarray, scale: float, n_past: int, raw: bool = False):
    x = np.ascontiguousarray(x, np.float32)
    out, ne = np.zeros_like(x), _ne(x.shape)
    rc = _lib().probe_scale_mask_softmax(dev.encode(), ne.ctypes.data, scale, n_past, x.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_scale_mask_softmax({dev}, {x.shape})", out)


# ------------------------------------------------------------------ case grids
def packed_nb3(t, pne):
    """(nb1, nb2, nb3) of a packed parent"""
    rb = row_bytes(t, pne[0])
    return rb, rb * pne[1], rb * pne[1] * pne[2]


def permuted(t, ne, seed=0) -> Source:
    """a view reading dims 1 and 2 of a packed parent [ne0, ne2, ne1, ne3] swapped (ggml_permute(p, 0, 2, 1, 3)), as `ne`"""
    pne = (ne[0], ne[2], ne[1], ne[3])
    nb1, nb2, nb3 = packed_nb3(t, pne)
    return Source(t, ne, parent_ne=pne, nb=(nb2, nb1, nb3), seed=seed)


def get_rows_grid():
    """(src, n ids per matrix, id order) per case: f32, f16 and every block format; rows of 96 and 4128 (32-element blocks, floats) or
    256 and 4352 (256-element blocks): neither a multiple of the 256-thread CTA but 256; src0 of 3 dims ([ne0, 5, 3], ids [n, 3]) and 4
    dims ([ne0, 4, 2, 2], ids [n, 2, 2]); random ids with repeats, descending and repeated ids"""
    out = []
    for k, t in enumerate((F32, F16) + BLOCK_TYPES):
        short, long_ = (256, 4352) if t in BLOCK_TYPES and orc().blck_size(t) == 256 else (96, 4128)
        out.append((block_source(t, (short, 9), seed=2 * k), 13, "random"))
        out.append((block_source(t, (long_, 5, 3), seed=2 * k + 1), 6, ("descending", "repeated")[k % 2]))
        if k % 4 == 0:
            out.append((block_source(t, (short, 4, 2, 2), seed=100 + k), 5, "random"))
    return out


def binary_grid():
    """(op, src0, src1, inplace, ggml_cpu_can): src1 broadcast along every subset of the four dims (each op four times); a src1 of half
    src0's ne0 (two whole repeats per row); src0 permuted, with padded rows, in place; src1 a strided view; src0 transposed (its ne0 not
    contiguous: ggml-cpu asserts nb00 == 4, so only the C ABI runs it)"""
    ne = (40, 5, 3, 2)
    out = []
    for m in range(16):
        ne1 = tuple(1 if m >> i & 1 else ne[i] for i in range(4))
        out.append((m % 4, Source(F32, ne, seed=m), Source(F32, ne1, seed=50 + m), False, True))
    for op in (ADD, MUL, SUB, DIV):
        out.append((op, Source(F32, ne, seed=20 + op), Source(F32, (20, 1, 3, 1), seed=70 + op), False, True))
        out.append((op, permuted(F32, ne, seed=24 + op), Source(F32, (40, 5, 1, 1), seed=74 + op), False, True))
        out.append((op, Source(F32, ne, parent_ne=(44, 5, 3, 2), seed=28 + op), Source(F32, (40, 1, 3, 1), seed=78 + op), True, True))
        out.append((op, Source(F32, ne, seed=32 + op), Source(F32, (40, 5, 1, 1), parent_ne=(48, 6, 1, 1), offs=16, seed=82 + op), False,
                    True))
        out.append((op, Source(F32, (5, 40, 3, 2), transpose=True, seed=36 + op), Source(F32, (40, 1, 1, 1), seed=86 + op), False, False))
    return out


NORM_NE0 = (1, 31, 32, 33, 255, 256, 257, 1023, 1024, 4096, 14336)


def norm_grid():
    """(rms, eps, src, offset, zero_rows): every row length of NORM_NE0 (either side of the launcher's 32 / 128 / 256-thread steps) for
    both norms, eps 1e-6 and 0, offsets 0 .. 1e4, strided rows (a padded parent), all-zero rows"""
    out = []
    for k, n in enumerate(NORM_NE0):
        rows = max(2, min(12, 65536 // n))
        for rms in (False, True):
            out.append((rms, 1e-6, Source(F32, (n, rows, 1, 1), seed=k), 0.0, False))
        out.append((False, 1e-6, Source(F32, (n, rows, 1, 1), seed=20 + k), (30.0, 1e3, 1e4)[k % 3], False))
        out.append((k % 2 == 1, 0.0, Source(F32, (n, 3, 2, 1), parent_ne=(n + 5, 3, 2, 1), seed=40 + k), 1.0, False))
    for rms in (False, True):
        for eps in (0.0, 1e-6):
            out.append((rms, eps, Source(F32, (64, 6, 1, 1), seed=60), 0.0, True))
    return out


def cpy_grid():
    """(op, src, dst): f32 -> f16, f16 -> f32 and f16 -> f16 copies from packed, permuted and transposed sources into packed and padded
    destination views at an offset; CONT of transposed and DUP of permuted sources (op 0 CPY, 1 CONT, 2 DUP)"""
    out = []
    ne = (37, 5, 3, 1)
    for k, (ts, td) in enumerate(((F32, F16), (F16, F32), (F16, F16), (F32, F32))):
        es = ES[td]
        out.append((0, Source(ts, ne, seed=k), Source(td, ne)))
        out.append((0, permuted(ts, ne, seed=10 + k), Source(td, ne, parent_ne=(40, 6, 3, 1), nb=(40 * es, 240 * es, 720 * es), offs=41 * es)))
        out.append((0, Source(ts, (5, 37, 3, 1), transpose=True, seed=20 + k), Source(td, ne)))
    for k, t in enumerate((F32, F16)):
        out.append((1, Source(t, (5, 37, 3, 1), transpose=True, seed=30 + k), None))
        out.append((2, permuted(t, ne, seed=32 + k), None))
    return out
