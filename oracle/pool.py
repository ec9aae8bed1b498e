"""TEST INFRASTRUCTURE ONLY: GGML_OP_POOL_2D, GGML_OP_UPSCALE, GGML_OP_LEAKY_RELU and GGML_OP_REPEAT cases and the reference's ops through
oracle/_ref/libggml_pool_probe.so (oracle/pool_probe.cpp).

`Source` describes a node's input (type, the parent tensor it is a view of, the view's ne / nb / offset, optionally transposed) and makes
its parent's bytes from a seed, with NaN, infinities and signed zeros among the values (raw words for REPEAT, NaN payloads included).
`PoolCase`, `UpscaleCase`, `LeakyCase` and `RepeatCase` describe one node each; `*_grid()` are the sets the CPU (host-compiled
b200_pool.cuh) and GPU (device kernel) parity tests run.  `pool_2d(dev, case)` etc. evaluate on a named ggml device ("CPU": ggml-cpu;
"B2000": the plug-in, once loaded with oracle.Ref().load_backend)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from .probe import probe_lib, result

F32, F16, I16, I32, BF16 = 0, 1, 25, 26, 30
ES = {F32: 4, I32: 4, F16: 2, BF16: 2, I16: 2}
POOL_MAX, POOL_AVG = 0, 1


def packed_nb(ne, es):
    nb = [es]
    for i in range(3):
        nb.append(nb[-1] * ne[i])
    return tuple(nb)


def pool_out_size(ins, ks, s, p):
    """ggml_calc_pool_output_size: in float, from the float padding"""
    f = np.float32
    return int((f(ins) + f(2) * f(p) - f(ks)) / f(s) + f(1))


@dataclass
class Source:
    """a node's input: view ne (ggml order) of a parent of shape parent_ne, strides nb1..nb3 in bytes (nb0 = the element size), byte
    offset offs; transpose: the node reads it through ggml_transpose (dims 0 and 1 swapped)"""
    type: int
    ne: tuple
    parent_ne: tuple | None = None
    nb: tuple | None = None              # (nb1, nb2, nb3); None: the parent's own
    offs: int = 0
    transpose: bool = False
    seed: int = 0

    def __post_init__(self):
        self.ne = tuple(self.ne) + (1,) * (4 - len(self.ne))
        self.parent_ne = tuple(self.parent_ne or self.ne) + (1,) * (4 - len(self.parent_ne or self.ne))
        if self.nb is None:
            self.nb = packed_nb(self.parent_ne, ES[self.type])[1:]

    def spec(self) -> np.ndarray:
        return np.array([self.type, *self.parent_ne, *self.ne, *self.nb, self.offs, int(self.transpose)], dtype=np.int64)

    def parent(self) -> np.ndarray:
        """the parent's elements, ggml dims reversed: f32 values with NaN / +-inf / -0 / ties among them; raw words for the other types"""
        rng = np.random.default_rng(15000 + self.seed)
        shape = self.parent_ne[::-1]
        if self.type == F32:
            x = (rng.standard_normal(shape) * 2.0).astype(np.float32)
            flat = x.reshape(-1)
            flat[3::23] = np.nan
            flat[5::29] = np.inf
            flat[7::31] = -np.inf
            flat[11::19] = -0.0
            flat[13::17] = 0.0
            flat[2::37] = flat[1::37][: len(flat[2::37])]            # equal neighbours: MAX ties
            return x
        es = ES[self.type]
        words = rng.integers(0, 1 << (8 * es), size=shape, dtype=np.uint64).astype(np.uint32 if es == 4 else np.uint16)
        flat = words.reshape(-1)
        flat[3::13] = 0x7fc01234 if es == 4 else 0x7e05           # NaN payloads (f32 / f16 / bf16 readings)
        flat[5::17] = 0x7f800001 if es == 4 else 0x7c01            # signalling NaNs
        flat[7::19] = 0x80000000 if es == 4 else 0x8000            # -0
        return words

    def view(self) -> tuple:
        """(ne, nb) through which the node reads the parent's bytes from offs, transposition applied"""
        nb = (ES[self.type],) + tuple(self.nb)
        if self.transpose:
            return (self.ne[1], self.ne[0], self.ne[2], self.ne[3]), (nb[1], nb[0], nb[2], nb[3])
        return self.ne, nb


@dataclass
class PoolCase:
    src: Source
    op: int
    k0: int
    k1: int
    s0: int
    s1: int
    p0: float = 0.0
    p1: float = 0.0

    @property
    def params(self):
        return (self.op, self.k0, self.k1, self.s0, self.s1, int(self.p0), int(self.p1))

    @property
    def ne_dst(self):
        ne, _ = self.src.view()
        return (pool_out_size(ne[0], self.k0, self.s0, self.p0), pool_out_size(ne[1], self.k1, self.s1, self.p1), ne[2], ne[3])

    def __str__(self):
        return (f"pool_2d {'max' if self.op == POOL_MAX else 'avg'} x={self.src.ne}/{self.src.parent_ne} k=({self.k0},{self.k1}) "
                f"s=({self.s0},{self.s1}) p=({self.p0},{self.p1})")


@dataclass
class UpscaleCase:
    src: Source
    ne_dst: tuple

    def __str__(self):
        return f"upscale x={self.src.ne}{'^T' if self.src.transpose else ''} -> {self.ne_dst}"


@dataclass
class LeakyCase:
    src: Source
    slope: float
    inplace: bool = False

    def __str__(self):
        return f"leaky_relu x={self.src.ne}/{self.src.parent_ne} slope={self.slope}{' inplace' if self.inplace else ''}"


@dataclass
class RepeatCase:
    src: Source
    ne_dst: tuple

    def __str__(self):
        return f"repeat type={self.src.type} x={self.src.ne}/{self.src.parent_ne} -> {self.ne_dst}"


def pool_grid() -> list:
    """MAX and AVG; windows 1-3, strides 1-3, paddings 0-2 (p >= k: windows wholly in the padding) on three input layouts (packed, rows
    padded beyond 4 ne0, rows and planes padded), two images; the 0.5-padding k2 s1 pool of YOLO"""
    out, i = [], 0
    for op in (POOL_MAX, POOL_AVG):
        for k in (1, 2, 3):
            for s in (1, 2, 3):
                for p in (0, 1, 2):
                    view = i % 3
                    ne = (9, 7, 3, 2)
                    if view == 0:
                        src = Source(F32, ne, seed=i)
                    elif view == 1:
                        src = Source(F32, ne, parent_ne=(14, 7, 3, 2), seed=i)
                    else:
                        src = Source(F32, ne, parent_ne=(12, 9, 3, 2), seed=i)
                    k1, s1, p1 = 1 + (k + i) % 3, 1 + (s + 1) % 3, (p + 1) % 3
                    out.append(PoolCase(src, op, k, k1, s, s1, p, p1))
                    i += 1
    for op in (POOL_MAX, POOL_AVG):
        out.append(PoolCase(Source(F32, (13, 13, 8, 1), seed=100 + op), op, 2, 2, 1, 1, 0.5, 0.5))
        out.append(PoolCase(Source(F32, (26, 26, 4, 2), seed=102 + op), op, 2, 2, 2, 2, 0, 0))
    return out


def upscale_grid() -> list:
    """integer factors, fractional ggml_upscale_ext factors (test-backend-ops' {2,5,7,11} -> {5,7,11,13}), strided and transposed inputs"""
    return [
        UpscaleCase(Source(F32, (7, 5, 3, 2), seed=1), (14, 10, 3, 2)),
        UpscaleCase(Source(F32, (4, 3, 2, 1), seed=2), (12, 9, 2, 1)),
        UpscaleCase(Source(F32, (2, 5, 7, 11), seed=3), (5, 7, 11, 13)),
        UpscaleCase(Source(F32, (5, 3, 2, 1), seed=4), (7, 8, 3, 2)),
        UpscaleCase(Source(F32, (6, 5, 3, 1), parent_ne=(9, 5, 3, 1), seed=5), (12, 10, 3, 1)),
        UpscaleCase(Source(F32, (5, 7, 3, 1), transpose=True, seed=6), (14, 10, 3, 1)),
    ]


def leaky_grid() -> list:
    """slopes 0.1, 0 and 1, in place and not, packed and padded rows"""
    out = []
    for i, slope in enumerate((0.1, 0.0, 1.0)):
        out.append(LeakyCase(Source(F32, (10, 5, 4, 3), seed=20 + i), slope))
        out.append(LeakyCase(Source(F32, (10, 5, 4, 3), seed=23 + i), slope, inplace=True))
    out.append(LeakyCase(Source(F32, (10, 5, 4, 1), parent_ne=(13, 5, 4, 1), seed=26), 0.1))
    return out


def repeat_grid() -> list:
    """every type ggml-cpu repeats, whole repeats along each dim, a strided src, the batch norm's [1, 1, C, 1] -> [W, H, C, N]"""
    out = []
    for i, t in enumerate((F32, I32, F16, BF16, I16)):
        out.append(RepeatCase(Source(t, (3, 2, 4, 1), seed=30 + i), (6, 4, 8, 2)))
        out.append(RepeatCase(Source(t, (3, 2, 4, 2), parent_ne=(5, 3, 4, 2), seed=35 + i), (3, 4, 4, 4)))
    out.append(RepeatCase(Source(F32, (1, 1, 16, 1), seed=40), (13, 11, 16, 2)))
    out.append(RepeatCase(Source(F32, (10, 5, 4, 2), seed=41), (10, 5, 4, 2)))
    return out


# ------------------------------------------------------------------ the probe
SIGNATURES = {
    "probe_pool_2d": [C.c_char_p, C.c_void_p] + [C.c_int] * 5 + [C.c_float] * 2 + [C.c_void_p, C.c_void_p],
    "probe_upscale": [C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
    "probe_leaky_relu": [C.c_char_p, C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_void_p],
    "probe_repeat": [C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
}


def _lib():
    return probe_lib("pool", "make -C oracle -f yolo.mk yolo", SIGNATURES)


def _dtype(t):
    return np.float32 if t == F32 else np.uint32 if ES[t] == 4 else np.uint16


def nbytes(ne, nb, es):
    """ggml_nbytes of a tensor with these extents and strides"""
    return es + sum((n - 1) * b for n, b in zip(ne, nb))


def pool_2d(dev: str, case: PoolCase, parent=None, raw: bool = False):
    """POOL_2D of `case` on `dev`: f32, ggml dims reversed"""
    L = _lib()
    parent = case.src.parent() if parent is None else parent
    out = np.zeros(case.ne_dst[::-1], dtype=np.float32)
    rc = L.probe_pool_2d(dev.encode(), case.src.spec().ctypes.data, case.op, case.k0, case.k1, case.s0, case.s1, case.p0, case.p1,
                         parent.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_pool_2d({dev}, {case})", out)


def upscale(dev: str, case: UpscaleCase, parent=None, raw: bool = False):
    L = _lib()
    parent = case.src.parent() if parent is None else parent
    out = np.zeros(tuple(case.ne_dst)[::-1], dtype=np.float32)
    ne = np.array(case.ne_dst, dtype=np.int64)
    rc = L.probe_upscale(dev.encode(), case.src.spec().ctypes.data, ne.ctypes.data, parent.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_upscale({dev}, {case})", out)


def leaky_relu(dev: str, case: LeakyCase, parent=None, raw: bool = False):
    """LEAKY_RELU of `case` on `dev`: not in place, the packed result (ggml dims reversed); in place, the bytes of the source view (its
    ggml_nbytes from its first element), as f32"""
    L = _lib()
    parent = case.src.parent() if parent is None else parent
    ne, nb = case.src.view()
    out = np.zeros(ne[::-1], dtype=np.float32) if not case.inplace else np.zeros(nbytes(ne, nb, 4) // 4, dtype=np.float32)
    rc = L.probe_leaky_relu(dev.encode(), case.src.spec().ctypes.data, case.slope, int(case.inplace), parent.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_leaky_relu({dev}, {case})", out)


def repeat(dev: str, case: RepeatCase, parent=None, raw: bool = False):
    """REPEAT of `case` on `dev`: raw words (uint32 / uint16), ggml dims reversed"""
    L = _lib()
    parent = case.src.parent() if parent is None else parent
    out = np.zeros(tuple(case.ne_dst)[::-1], dtype=_dtype(case.src.type) if case.src.type != F32 else np.uint32)
    ne = np.array(case.ne_dst, dtype=np.int64)
    rc = L.probe_repeat(dev.encode(), case.src.spec().ctypes.data, ne.ctypes.data, parent.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_repeat({dev}, {case})", out)
