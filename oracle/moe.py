"""TEST INFRASTRUCTURE ONLY: GGML_OP_ARGSORT / GGML_OP_SUM_ROWS cases and the reference's ops through oracle/_ref/libggml_moe_probe.so
(oracle/moe_probe.cpp).

`Case` describes one node's source (shape, row kind, strided view); `argsort_grid()` is the set the CPU (host-compiled sort network) and
GPU (device kernel) parity tests run; `argsort(dev, case, order)` / `sum_rows(dev, case)` evaluate a case on a named ggml device ("CPU":
ggml-cpu; "B2000": the plug-in, once loaded with oracle.Ref().load_backend).  The checks of a sorted row live here too, so the host and
device tests apply the same rules."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import oracle as O

ASC, DESC = 0, 1
KINDS = ("tiefree", "ties", "special")
ARGSORT_LENGTHS = (1, 2, 7, 8, 16, 60, 64, 128, 255, 1000, 1024)


@dataclass
class Case:
    ne: tuple                     # (ne0, ne1, ne2, ne3) of the node's source
    kind: str = "tiefree"         # tiefree: distinct values; ties: a few values, +-0 among them; special: +-inf and NaNs among normals
    view: int = 0                 # 0 contiguous; 1 rows padded by 3 floats (evenly spaced); 2 corner of a [2 ne0, 2 ne1, 3 ne2, ne3] parent
    seed: int = 0

    @property
    def parent_ne(self) -> tuple:
        ne0, ne1, ne2, ne3 = self.ne
        return {0: self.ne, 1: (ne0 + 3, ne1, ne2, ne3), 2: (ne0 * 2, ne1 * 2, ne2 * 3, ne3)}[self.view]

    def parent(self) -> np.ndarray:
        """the parent tensor's elements in ggml order, as a numpy array of shape parent_ne reversed"""
        rng = np.random.default_rng(5000 + self.seed)
        shape = self.parent_ne[::-1]
        n = int(np.prod(shape))
        if self.kind == "tiefree":
            # distinct per row: a random permutation of a spread of values of both signs (distinct over the whole tensor as well)
            x = (rng.permutation(n).astype(np.float64) - n / 2.0) * 0.37
        elif self.kind == "ties":
            x = rng.choice(np.array([-1.5, -0.0, 0.0, 0.25, 0.25, 3.0]), n)
        else:
            x = rng.standard_normal(n)
            specials = np.array([np.inf, -np.inf, np.nan, -np.nan], dtype=np.float32)
            x = x.astype(np.float32)
            pick = rng.random(n) < 0.2
            x[pick] = rng.choice(specials, int(pick.sum()))
            bits = x.view(np.uint32)
            odd = np.isnan(x) & (rng.random(n) < 0.5)
            bits[odd] |= 0x1234                                      # NaNs with other payloads
            return x.reshape(shape)
        return x.astype(np.float32).reshape(shape)

    def rows(self, parent: np.ndarray | None = None) -> np.ndarray:
        """the node's source as contiguous rows [ne1 * ne2 * ne3, ne0]"""
        p = self.parent() if parent is None else parent
        ne0, ne1, ne2, ne3 = self.ne
        return np.ascontiguousarray(p[:ne3, :ne2, :ne1, :ne0]).reshape(-1, ne0)

    def __str__(self):
        return f"ne={self.ne} kind={self.kind} view={self.view}"


def argsort_grid(strided: bool = False) -> list:
    """every length of ARGSORT_LENGTHS x the three row kinds, three rows each; strided: in addition strided (evenly spaced) and
    multi-dimensional sources"""
    out, seed = [], 0
    for n in ARGSORT_LENGTHS:
        for kind in KINDS:
            seed += 1
            out.append(Case((n, 3, 1, 1), kind, seed=seed))
            if strided:
                out.append(Case((n, 3, 2, 2), kind, view=1, seed=seed + 1000))
    return out


def check_sorted_row(x: np.ndarray, got: np.ndarray, order: int, want: np.ndarray | None = None) -> None:
    """the device / emulated rule on one row: a permutation; numbers in order (ties in ascending index, -0 == +0) before every NaN;
    when `want` (ggml-cpu's row) is given and the row holds no NaN, the same sequence of values, and on a tie-free row the same indices"""
    n = x.size
    assert np.array_equal(np.sort(got), np.arange(n)), "not a permutation"
    v = x[got].astype(np.float64)
    nan = np.isnan(v)
    k = int((~nan).sum())
    assert not nan[:k].any(), "a NaN sorts before a number"
    num = v[:k] if order == ASC else -v[:k]
    assert np.all(num[1:] >= num[:-1]), "numbers out of order"                # (not np.diff: inf - inf is NaN)
    eq = num[1:] == num[:-1]
    assert np.all(np.diff(got[:k])[eq] > 0), "ties not in ascending index"
    if want is not None and not np.isnan(x).any():
        assert np.array_equal(x[want].astype(np.float64), v), "value sequence differs from ggml-cpu's"
        if np.unique(x).size == n:
            assert np.array_equal(got, want), "indices differ from ggml-cpu's on a tie-free row"


_lib = None


def _probe_lib():
    global _lib
    if _lib is None:
        O.Ref()                                            # loads the reference libraries (and the shared backend registry) globally
        so = O.REF_DIR / "libggml_moe_probe.so"
        if not so.exists():
            raise RuntimeError(f"{so} missing (make -C oracle -f moe.mk moe where the reference tree exists)")
        L = C.CDLL(str(so))
        L.probe_argsort.restype = C.c_int
        L.probe_argsort.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.probe_sum_rows.restype = C.c_int
        L.probe_sum_rows.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def argsort(dev: str, case: Case, order: int, parent: np.ndarray | None = None, raw: bool = False):
    """ARGSORT of `case` on ggml device `dev`: i32 rows [ne1 * ne2 * ne3, ne0].  raw: return the probe's code instead of raising"""
    L = _probe_lib()
    x = np.ascontiguousarray(case.parent() if parent is None else parent, dtype=np.float32)
    ne = np.array(case.ne, dtype=np.int64)
    out = np.empty(int(np.prod(case.ne)), dtype=np.int32)
    rc = L.probe_argsort(dev.encode(), ne.ctypes.data, case.view, order, x.ctypes.data, out.ctypes.data)
    if raw:
        return rc
    if rc != 0:
        raise RuntimeError(f"probe_argsort({dev}, {case}, {order}) returned {rc}")
    return out.reshape(-1, case.ne[0])


def sum_rows(dev: str, case: Case, parent: np.ndarray | None = None) -> np.ndarray:
    """SUM_ROWS of `case` on ggml device `dev`: f32 [ne1 * ne2 * ne3]"""
    L = _probe_lib()
    x = np.ascontiguousarray(case.parent() if parent is None else parent, dtype=np.float32)
    ne = np.array(case.ne, dtype=np.int64)
    out = np.empty(int(np.prod(case.ne[1:])), dtype=np.float32)
    rc = L.probe_sum_rows(dev.encode(), ne.ctypes.data, case.view, x.ctypes.data, out.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"probe_sum_rows({dev}, {case}) returned {rc}")
    return out
