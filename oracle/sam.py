"""TEST INFRASTRUCTURE ONLY: GGML_OP_WIN_PART, GGML_OP_WIN_UNPART, GGML_OP_GET_REL_POS, GGML_OP_ADD_REL_POS, GGML_OP_CONV_TRANSPOSE_2D,
GGML_OP_SIN and GGML_OP_COS cases and the reference's ops through oracle/_ref/libggml_sam_probe.so (oracle/sam_probe.cpp).

Sources are oracle/pool.py's `Source` (type, the parent tensor it is a view of, the view's ne / nb / offset), whose parents carry NaN,
infinities and signed zeros (raw words for f16).  `WinPartCase`, `WinUnpartCase`, `RelPosCase`, `AddRelPosCase`, `ConvT2dCase` and
`SinCosCase` describe one node each; `*_grid()` are the sets the CPU (host-compiled b200_sam.cuh) and GPU (device kernel) parity tests run.
`win_part(dev, case)` etc. evaluate on a named ggml device ("CPU": ggml-cpu; "B2000": the plug-in, once loaded with
oracle.Ref().load_backend)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import oracle as O
from .pool import F16, F32, Source, _result

SIN, COS = 0, 1


def cdiv(a, b):
    return -(-a // b)


@dataclass
class WinPartCase:
    src: Source          # f32 [C, W0, H0, 1]
    w: int

    @property
    def ne_dst(self):
        c, w0, h0, _ = self.src.ne
        return (c, self.w, self.w, cdiv(w0, self.w) * cdiv(h0, self.w))

    def __str__(self):
        return f"win_part x={self.src.ne}/{self.src.parent_ne} w={self.w}"


@dataclass
class WinUnpartCase:
    src: Source          # f32 [C, w, w, np]
    w0: int
    h0: int
    w: int

    @property
    def ne_dst(self):
        return (self.src.ne[0], self.w0, self.h0, 1)

    def __str__(self):
        return f"win_unpart x={self.src.ne}/{self.src.parent_ne} -> {self.w0}x{self.h0} w={self.w}"


@dataclass
class RelPosCase:
    src: Source          # f16 [C, 2w - 1]
    w: int

    @property
    def ne_dst(self):
        return (self.src.ne[0], self.w, self.w, 1)

    def __str__(self):
        return f"get_rel_pos x={self.src.ne}/{self.src.parent_ne} w={self.w}"


@dataclass
class AddRelPosCase:
    """a f32 [L L, A B, P, n3], pw and ph f32 [L, A, B, P]; values with exponents over a wide range, so that the two orders of the adds give
    different bits for many elements, plus NaN / +-inf / -0 (Source's specials) in a"""
    L: int
    A: int
    B: int
    P: int
    inplace: bool = False
    seed: int = 0
    n3: int = 1
    a_parent_ne: tuple | None = None         # a view of a larger parent (a layout ggml-cpu reads differently)

    def sources(self):
        ne = (self.L * self.L, self.A * self.B, self.P, self.n3)
        pne = (self.L, self.A, self.B, self.P)
        return (Source(F32, ne, parent_ne=self.a_parent_ne, seed=3000 + self.seed),
                Source(F32, pne, seed=3100 + self.seed), Source(F32, pne, seed=3200 + self.seed))

    def parents(self):
        """a (with Source's specials), pw, ph: the three scaled differently, so that rounding the two sums differently is common"""
        a, pw, ph = (s.parent() for s in self.sources())
        rng = np.random.default_rng(3300 + self.seed)
        pw = (pw * np.exp2(rng.integers(-3, 3, pw.shape)).astype(np.float32)).astype(np.float32)
        ph = (ph * np.exp2(rng.integers(-3, 3, ph.shape)).astype(np.float32)).astype(np.float32)
        np.nan_to_num(pw, copy=False, nan=1.5, posinf=3.25, neginf=-3.25)
        np.nan_to_num(ph, copy=False, nan=-0.75, posinf=2.5, neginf=-2.5)
        return a, pw, ph

    @property
    def ne_dst(self):
        return (self.L * self.L, self.A * self.B, self.P, self.n3)

    def __str__(self):
        return f"add_rel_pos L={self.L} A={self.A} B={self.B} P={self.P}{' inplace' if self.inplace else ''}"


def add_rel_pos_numpy(a, pw, ph, L, order="ggml"):
    """ADD_REL_POS in numpy, f32, a [P, A B, L L] and pw / ph [P, B, A, L] (torch order).  order "ggml": ph first where kh <= kw (ggml-cpu's
    loop, ggml-cpu.c:11823-11840); "pw": pw first everywhere; "ph": ph first everywhere"""
    P, Q = a.shape[0], a.shape[1]
    x = a.reshape(P, Q, L, L)                                        # [.., kh, kw]
    h = ph.reshape(P, Q, L)[:, :, :, None].astype(np.float32)        # ph[r, kh]
    w = pw.reshape(P, Q, L)[:, :, None, :].astype(np.float32)        # pw[r, kw]
    with np.errstate(invalid="ignore", over="ignore"):
        h_first = (x + h) + w
        w_first = (x + w) + h
    if order == "ph":
        return h_first.reshape(a.shape)
    if order == "pw":
        return w_first.reshape(a.shape)
    kh = np.arange(L)[:, None]
    kw = np.arange(L)[None, :]
    return np.where(kh <= kw, h_first, w_first).reshape(a.shape)


@dataclass
class ConvT2dCase:
    """kernel f16 [Kw, Kh, Cout, Cin], input f32 [W, H, Cin, n]; values ~ N(0, 1) (kernel scaled by 1/sqrt(Cin)); specials: NaN, +-inf and
    -0 among the input values"""
    Cin: int
    Cout: int
    Kw: int
    Kh: int
    W: int
    H: int
    s: int
    seed: int = 0
    k_parent_ne: tuple | None = None         # kernel planes in a larger parent (nb1 / nb2 / nb3 padded)
    x_parent_ne: tuple | None = None         # input rows / channels in a larger parent
    specials: bool = False
    n: int = 1

    def sources(self):
        return (Source(F16, (self.Kw, self.Kh, self.Cout, self.Cin), parent_ne=self.k_parent_ne),
                Source(F32, (self.W, self.H, self.Cin, self.n), parent_ne=self.x_parent_ne))

    def parents(self):
        ks, xs = self.sources()
        rng = np.random.default_rng(4000 + self.seed)
        k = (rng.standard_normal(ks.parent_ne[::-1]) / np.sqrt(max(self.Cin, 1))).astype(np.float16)
        x = rng.standard_normal(xs.parent_ne[::-1]).astype(np.float32)
        if self.specials:
            f = x.reshape(-1)
            f[3::97] = np.nan
            f[5::89] = np.inf
            f[7::83] = -np.inf
            f[11::19] = -0.0
            f[13::23] = 70000.0                      # beyond f16: rounds to inf
        return k, x

    @property
    def ne_dst(self):
        return ((self.W - 1) * self.s + self.Kw, (self.H - 1) * self.s + self.Kh, self.Cout, self.n)

    def __str__(self):
        return (f"conv_transpose_2d Cin={self.Cin} Cout={self.Cout} k={self.Kw}x{self.Kh} in={self.W}x{self.H} s={self.s}"
                f"{' specials' if self.specials else ''}{' strided' if self.k_parent_ne or self.x_parent_ne else ''}")


def conv_transpose_2d_reference(case: ConvT2dCase, k, x):
    """f64 CONV_TRANSPOSE_2D of the fp16-rounded operands (first image): [Cout, OH, OW]"""
    ks, xs = case.sources()
    kk = k[: case.Cin, : case.Cout, : case.Kh, : case.Kw].astype(np.float64)                      # [Cin, Cout, Kh, Kw]
    xx = x[0, : case.Cin, : case.H, : case.W].astype(np.float16).astype(np.float64)               # [Cin, H, W]
    OW, OH = case.ne_dst[0], case.ne_dst[1]
    out = np.zeros((case.Cout, OH, OW))
    for ky in range(case.Kh):
        for kx in range(case.Kw):
            t = np.einsum("chw,co->ohw", xx, kk[:, :, ky, kx])
            out[:, ky: ky + (case.H - 1) * case.s + 1: case.s, kx: kx + (case.W - 1) * case.s + 1: case.s] += t
    return out


@dataclass
class SinCosCase:
    src: Source
    op: int

    def __str__(self):
        return f"{'sin' if self.op == SIN else 'cos'} x={self.src.ne}"


def sin_cos_parent(case: SinCosCase):
    """arguments over [-1e4, 1e4] on a log scale (both signs), the SAM range 2 pi [-3, 3], and NaN / +-inf / +-0"""
    rng = np.random.default_rng(5000 + case.src.seed)
    n = int(np.prod(case.src.parent_ne))
    x = np.empty(n, np.float32)
    half = n // 2
    x[:half] = (np.sign(rng.standard_normal(half)) * np.exp(rng.uniform(np.log(1e-6), np.log(1e4), half))).astype(np.float32)
    x[half:] = rng.uniform(-6 * np.pi, 6 * np.pi, n - half).astype(np.float32)
    x[3::101] = np.nan
    x[5::103] = np.inf
    x[7::107] = -np.inf
    x[11::109] = -0.0
    x[13::113] = 0.0
    return x.reshape(case.src.parent_ne[::-1])


def ulp_error(got, x):
    """|got - f(x) in f64| in units of the f32 spacing at the f64 value, for sin / cos of f32 x; NaN where the f64 value is NaN"""
    return np.abs(got.astype(np.float64) - x) / np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


# ------------------------------------------------------------------ grids
def win_grid():
    """(C, W0, H0, w): windows that divide the image, ones that do not (padding on one or both sides), w = 1, w beyond the image, the SAM
    window 14 on a 32 x 32 image"""
    return [(3, 8, 8, 4), (5, 9, 7, 4), (4, 7, 5, 1), (2, 5, 6, 7), (6, 32, 32, 14), (7, 14, 28, 14), (33, 10, 3, 3)]


def win_part_grid():
    return [WinPartCase(Source(F32, (c, w0, h0, 1), seed=i), w) for i, (c, w0, h0, w) in enumerate(win_grid())]


def win_unpart_grid():
    out = []
    for i, (c, w0, h0, w) in enumerate(win_grid()):
        np_ = cdiv(w0, w) * cdiv(h0, w)
        out.append(WinUnpartCase(Source(F32, (c, w, w, np_), seed=20 + i), w0, h0, w))
    out.append(WinUnpartCase(Source(F32, (5, 4, 4, 9), seed=40), 9, 7, 4))          # more windows than the image needs: the last is ignored
    return out


def rel_pos_grid():
    """w = 1 .. 64, C from 1 to 12 (odd and even row lengths)"""
    return [RelPosCase(Source(F16, (1 + (w * 5) % 12, 2 * w - 1), seed=100 + w), w) for w in range(1, 65)]


def add_rel_pos_grid():
    """L = 1, 2, 7, 14 (query grids L x L and others), in place and not"""
    out = []
    for i, (L, A, B, P) in enumerate([(1, 3, 1, 16), (2, 2, 2, 3), (7, 7, 7, 2), (14, 14, 14, 2), (7, 3, 5, 1), (2, 5, 1, 4)]):
        out.append(AddRelPosCase(L, A, B, P, inplace=False, seed=i))
        out.append(AddRelPosCase(L, A, B, P, inplace=True, seed=10 + i))
    return out


def conv_transpose_grid():
    """s < K, s = K, s > K; Cin = 1; Cin and Cout not multiples of the device tile (32); Kw != Kh; strided kernel planes and input rows;
    NaN / +-inf / -0 inputs"""
    return [ConvT2dCase(4, 5, 3, 3, 6, 5, 2, seed=0), ConvT2dCase(16, 8, 2, 2, 7, 6, 2, seed=1), ConvT2dCase(3, 4, 2, 2, 5, 4, 3, seed=2),
            ConvT2dCase(1, 3, 3, 3, 5, 5, 1, seed=3), ConvT2dCase(40, 37, 2, 2, 9, 8, 2, seed=4), ConvT2dCase(70, 33, 3, 2, 5, 3, 2, seed=5),
            ConvT2dCase(5, 6, 1, 1, 4, 3, 4, seed=6), ConvT2dCase(9, 7, 4, 3, 35, 3, 3, seed=7),
            ConvT2dCase(6, 5, 3, 3, 6, 5, 2, seed=8, k_parent_ne=(3, 3, 6, 6), x_parent_ne=(8, 6, 6, 1)),
            ConvT2dCase(8, 9, 2, 2, 6, 5, 2, seed=9, specials=True)]


def sin_cos_grid():
    return [SinCosCase(Source(F32, (1000, 3, 1, 1), seed=i), op) for i, op in enumerate((SIN, COS))]


# ------------------------------------------------------------------ the probe
_lib = None


def _probe_lib():
    global _lib
    if _lib is None:
        O.Ref()                                            # loads the reference libraries (and the shared backend registry) globally
        so = O.REF_DIR / "libggml_sam_probe.so"
        if not so.exists():
            raise RuntimeError(f"{so} missing (make -C oracle -f sam.mk sam where the reference tree exists)")
        L = C.CDLL(str(so))
        vp, i = C.c_void_p, C.c_int
        for name, args in (("probe_win_part", [C.c_char_p, vp, i, vp, vp]), ("probe_win_unpart", [C.c_char_p, vp, i, i, i, vp, vp]),
                           ("probe_get_rel_pos", [C.c_char_p, vp, i, vp, vp]),
                           ("probe_add_rel_pos", [C.c_char_p, vp, vp, vp, i, vp, vp, vp, vp]),
                           ("probe_conv_transpose_2d", [C.c_char_p, vp, vp, i, vp, vp, vp]), ("probe_sin_cos", [C.c_char_p, vp, i, vp, vp])):
            fn = getattr(L, name)
            fn.restype, fn.argtypes = C.c_int, args
        _lib = L
    return _lib


def win_part(dev: str, case: WinPartCase, parent=None, raw: bool = False):
    """WIN_PART of `case` on `dev`: raw uint32 words, ggml dims reversed"""
    parent = case.src.parent() if parent is None else parent
    out = np.zeros(case.ne_dst[::-1], dtype=np.uint32)
    spec = case.src.spec()
    rc = _probe_lib().probe_win_part(dev.encode(), spec.ctypes.data, case.w, parent.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_win_part({dev}, {case})", out)


def win_unpart(dev: str, case: WinUnpartCase, parent=None, raw: bool = False):
    parent = case.src.parent() if parent is None else parent
    out = np.zeros(case.ne_dst[::-1], dtype=np.uint32)
    spec = case.src.spec()
    rc = _probe_lib().probe_win_unpart(dev.encode(), spec.ctypes.data, case.w0, case.h0, case.w, parent.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_win_unpart({dev}, {case})", out)


def get_rel_pos(dev: str, case: RelPosCase, parent=None, raw: bool = False):
    """GET_REL_POS of `case` on `dev`: raw uint16 words"""
    parent = case.src.parent() if parent is None else parent
    out = np.zeros(case.ne_dst[::-1], dtype=np.uint16)
    spec = case.src.spec()
    rc = _probe_lib().probe_get_rel_pos(dev.encode(), spec.ctypes.data, case.w, parent.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_get_rel_pos({dev}, {case})", out)


def add_rel_pos(dev: str, case: AddRelPosCase, parents=None, raw: bool = False):
    """ADD_REL_POS of `case` on `dev`: f32, ggml dims reversed (in place: the bytes of a's view, which is packed in every such case)"""
    a, pw, ph = case.parents() if parents is None else parents
    specs = [s.spec() for s in case.sources()]                     # held: the probe reads them through raw pointers
    out = np.zeros(case.ne_dst[::-1], dtype=np.float32)
    rc = _probe_lib().probe_add_rel_pos(dev.encode(), *(s.ctypes.data for s in specs), int(case.inplace),
                                        a.ctypes.data, pw.ctypes.data, ph.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_add_rel_pos({dev}, {case})", out)


def conv_transpose_2d(dev: str, case: ConvT2dCase, parents=None, raw: bool = False):
    """CONV_TRANSPOSE_2D of `case` on `dev`: f32 [n, Cout, OH, OW]"""
    k, x = case.parents() if parents is None else parents
    sk, sx = (s.spec() for s in case.sources())                    # held: the probe reads them through raw pointers
    out = np.zeros(case.ne_dst[::-1], dtype=np.float32)
    rc = _probe_lib().probe_conv_transpose_2d(dev.encode(), sk.ctypes.data, sx.ctypes.data, case.s, k.ctypes.data, x.ctypes.data,
                                              out.ctypes.data)
    return _result(rc, raw, f"probe_conv_transpose_2d({dev}, {case})", out)


def sin_cos(dev: str, case: SinCosCase, parent=None, raw: bool = False):
    parent = sin_cos_parent(case) if parent is None else parent
    out = np.zeros(case.src.ne[::-1], dtype=np.float32)
    spec = case.src.spec()
    rc = _probe_lib().probe_sin_cos(dev.encode(), spec.ctypes.data, case.op, parent.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_sin_cos({dev}, {case})", out)
