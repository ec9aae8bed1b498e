"""TEST INFRASTRUCTURE ONLY: GGML_OP_CONCAT / GGML_OP_SSM_CONV / GGML_OP_SSM_SCAN cases and the reference's ops through
oracle/_ref/libggml_ssm_probe.so (oracle/ssm_probe.cpp).

`ConcatCase`, `ConvCase` and `ScanCase` describe one node's sources (shapes, views, value kinds) and make their data from a seed;
`conv_grid()` / `scan_grid()` / `concat_grid()` are the sets the CPU (host-compiled b200_ssm.cuh) and GPU (device kernels) parity tests run;
`concat(dev, case)`, `ssm_conv(dev, case)` and `ssm_scan(dev, case)` evaluate a case on a named ggml device ("CPU": ggml-cpu; "B2000": the
plug-in, once loaded with oracle.Ref().load_backend).  `View` gives each source's parent array with the ne / nb / offset through which the
node reads it, exactly as ssm_probe.cpp's source() builds it, so the host emulation reads the same bytes."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from .probe import probe_lib, ptrs, result

F32, I32, F16 = 0, 1, 2
NP_TYPES = {F32: np.float32, I32: np.int32, F16: np.float16}


@dataclass
class View:
    """a node source: parent (numpy, ggml dims reversed) read as ne / nb (bytes) from byte offset `offs`"""
    parent: np.ndarray
    ne: tuple
    nb: tuple
    offs: int = 0


def _nb(shape_ggml, es):
    nb = [es]
    for i in range(3):
        nb.append(nb[-1] * shape_ggml[i])
    return tuple(nb)


def parent_ne(ne, view):
    """the parent shape ssm_probe.cpp's source() allocates for a source of shape ne through `view`"""
    ne0, ne1, ne2, ne3 = ne
    return {0: ne, 1: (ne0 * 2, ne1 * 4, ne2 * 3, ne3), 2: (ne1, ne0, ne2, ne3), 3: (ne0, ne1 + 3, ne2, ne3)}[view]


def make_view(parent: np.ndarray, ne, view) -> View:
    pnb = _nb(parent_ne(ne, view), parent.itemsize)
    if view == 2:
        return View(parent, tuple(ne), (pnb[1], pnb[0], pnb[2], pnb[3]))
    return View(parent, tuple(ne), pnb)


def read(v: View) -> np.ndarray:
    """the source as a contiguous array, ggml dims reversed"""
    flat = v.parent.reshape(-1).view(np.uint8)[v.offs:].view(v.parent.dtype)
    return np.lib.stride_tricks.as_strided(flat, shape=v.ne[::-1], strides=v.nb[::-1]).copy()


# ------------------------------------------------------------------ cases
@dataclass
class ConcatCase:
    type: int
    ne_a: tuple
    ne_b: tuple
    dim: int
    view_a: int = 0
    view_b: int = 0
    seed: int = 0

    @property
    def ne_dst(self):
        return tuple(self.ne_a[k] + (self.ne_b[k] if k == self.dim else 0) for k in range(4))

    def parents(self):
        rng = np.random.default_rng(7000 + self.seed)
        out = []
        for ne, view in ((self.ne_a, self.view_a), (self.ne_b, self.view_b)):
            shape = parent_ne(ne, view)[::-1]
            if self.type == I32:
                out.append(rng.integers(-(1 << 31), (1 << 31) - 1, shape, dtype=np.int64).astype(np.int32))
            else:
                x = rng.standard_normal(shape).astype(NP_TYPES[self.type])
                if self.type == F32:                                    # NaNs with payloads and -0.0 must come through bit for bit
                    x.reshape(-1).view(np.uint32)[::17] = 0x7FC01234
                    x.reshape(-1)[5::19] = -0.0
                out.append(x)
        return out

    def __str__(self):
        return f"concat type={self.type} a={self.ne_a}/v{self.view_a} b={self.ne_b}/v{self.view_b} dim={self.dim}"


@dataclass
class ConvCase:
    d_conv: int
    d_inner: int
    n_t: int
    n_s: int
    view_sx: int = 0            # 0 or 3 (rows packed, planes spread)
    view_c: int = 0             # 0 or 3 (rows packed: ggml-cpu reads row i1 of c at i1 * d_conv, whatever its nb1)
    seed: int = 0

    @property
    def ne_sx(self):
        return (self.d_conv - 1 + self.n_t, self.d_inner, self.n_s, 1)

    @property
    def ne_c(self):
        return (self.d_conv, self.d_inner, 1, 1)

    def views(self):
        rng = np.random.default_rng(8000 + self.seed)
        sx = rng.standard_normal(parent_ne(self.ne_sx, self.view_sx)[::-1]).astype(np.float32)
        c = (rng.standard_normal(parent_ne(self.ne_c, self.view_c)[::-1]) / np.sqrt(self.d_conv)).astype(np.float32)
        return make_view(sx, self.ne_sx, self.view_sx), make_view(c, self.ne_c, self.view_c)

    def __str__(self):
        return f"ssm_conv d_conv={self.d_conv} d_inner={self.d_inner} n_t={self.n_t} n_s={self.n_s} views={self.view_sx},{self.view_c}"


@dataclass
class ScanCase:
    d_state: int
    d_inner: int
    n_t: int
    n_s: int
    bc_rank: int = -1           # >= 0: B and C are views of one x_db [bc_rank + 2 d_state, n_t, n_s] (strided, as in the Mamba layer)
    seed: int = 0

    def views(self):
        """s, x, dt, A, B, C as Views (B and C share their parent when bc_rank >= 0)"""
        rng = np.random.default_rng(9000 + self.seed)
        ds, di, nt, ns = self.d_state, self.d_inner, self.n_t, self.n_s
        f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
        s = f(rng.standard_normal((ns, di, ds)))
        x = f(rng.standard_normal((ns, nt, di)))
        # dt: mostly where a trained model's pre-activations lie, plus values at and on both sides of the softplus cut-off at 20
        dt = rng.normal(-3.0, 2.5, (ns, nt, di))
        pick = rng.random(dt.shape)
        dt[pick < 0.10] = rng.uniform(20.0, 40.0, int((pick < 0.10).sum()))
        dt[(pick >= 0.10) & (pick < 0.15)] = rng.uniform(10.0, 20.0, int(((pick >= 0.10) & (pick < 0.15)).sum()))
        dt[(pick >= 0.15) & (pick < 0.17)] = 20.0
        dt = f(dt)
        A = f(-(np.arange(ds)[None, :] + 1.0) * rng.uniform(0.5, 2.0, (di, 1)))
        out = [View(s, (ds, di, ns, 1), _nb((ds, di, ns, 1), 4)), View(x, (di, nt, ns, 1), _nb((di, nt, ns, 1), 4)),
               View(dt, (di, nt, ns, 1), _nb((di, nt, ns, 1), 4)), View(A, (ds, di, 1, 1), _nb((ds, di, 1, 1), 4))]
        if self.bc_rank < 0:
            for _ in range(2):
                b = f(rng.standard_normal((ns, nt, ds)))
                out.append(View(b, (ds, nt, ns, 1), _nb((ds, nt, ns, 1), 4)))
        else:
            w = self.bc_rank + 2 * ds
            xdb = f(rng.standard_normal((ns, nt, w)))
            nb = _nb((w, nt, ns, 1), 4)
            out.append(View(xdb, (ds, nt, ns, 1), nb, 4 * self.bc_rank))
            out.append(View(xdb, (ds, nt, ns, 1), nb, 4 * (self.bc_rank + ds)))
        return out

    @property
    def n_y(self):
        return self.d_inner * self.n_t * self.n_s

    def __str__(self):
        return f"ssm_scan d_state={self.d_state} d_inner={self.d_inner} n_t={self.n_t} n_s={self.n_s} bc_rank={self.bc_rank}"


CONV_D_CONV, CONV_N_T, CONV_N_S = (2, 4, 8), (1, 5, 64), (1, 3)
SCAN_D_STATE, SCAN_N_T, SCAN_N_S = (1, 16, 64, 256), (1, 5, 64), (1, 3)


def conv_grid() -> list:
    """d_conv x n_t x n_s, d_inner 37; the views cycle through (packed, packed), (spread planes, c corner), (spread planes, packed)"""
    out, i = [], 0
    for dc in CONV_D_CONV:
        for nt in CONV_N_T:
            for ns in CONV_N_S:
                vs, vc = ((0, 0), (3, 3), (3, 0))[i % 3]
                out.append(ConvCase(dc, 37, nt, ns, vs, vc, seed=i))
                i += 1
    return out


def scan_grid() -> list:
    """d_state x n_t x n_s, d_inner 33; B and C strided views of an x_db for every other (d_state, n_t)"""
    out, i = [], 0
    for ds in SCAN_D_STATE:
        for nt in SCAN_N_T:
            for ns in SCAN_N_S:
                out.append(ScanCase(ds, 33, nt, ns, bc_rank=(5 if (i // 2) % 2 else -1), seed=i))
                i += 1
    return out


def concat_grid() -> list:
    """f32 and i32, every dim, contiguous / strided / transposed operands (the Mamba form: dim 0, b transposed)"""
    out, i = [], 0
    for t in (F32, I32):
        for dim in range(4):
            for va, vb in ((0, 0), (1, 0), (0, 1), (1, 1), (0, 2), (1, 2)):
                ne_a = (5, 6, 3, 2)
                ne_b = tuple(7 if k == dim else ne_a[k] for k in range(4))
                out.append(ConcatCase(t, ne_a, ne_b, dim, va, vb, seed=i))
                i += 1
    out.append(ConcatCase(F32, (3, 1536, 2, 1), (7, 1536, 2, 1), 0, 0, 2, seed=i))      # the Mamba layer's conv_x (d_conv 4, 7-token prompts)
    return out


# ------------------------------------------------------------------ the probe
SIGNATURES = {
    "probe_concat": [C.c_char_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p],
    "probe_ssm_conv": [C.c_char_p] + [C.c_int64] * 4 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p],
    "probe_ssm_scan": [C.c_char_p] + [C.c_int64] * 5 + [C.c_void_p, C.c_void_p],
}


def _lib():
    return probe_lib("ssm", "make -C oracle -f decoders.mk mamba", SIGNATURES)


def concat(dev: str, case: ConcatCase, raw: bool = False):
    """CONCAT of `case` on ggml device `dev`: the result, contiguous, ggml dims reversed.  raw: return the probe's code"""
    L = _lib()
    parents = case.parents()
    out = np.zeros(case.ne_dst[::-1], dtype=NP_TYPES[case.type])
    ne_a, ne_b = np.array(case.ne_a, dtype=np.int64), np.array(case.ne_b, dtype=np.int64)
    rc = L.probe_concat(dev.encode(), case.type, ne_a.ctypes.data, case.view_a, ne_b.ctypes.data, case.view_b, case.dim, ptrs(parents), out.ctypes.data)
    return result(rc, raw, f"probe_concat({dev}, {case})", out)


def ssm_conv(dev: str, case: ConvCase, views=None, raw: bool = False):
    """SSM_CONV of `case` on `dev`: f32 [n_s, n_t, d_inner]"""
    L = _lib()
    sx, c = views or case.views()
    out = np.zeros((case.n_s, case.n_t, case.d_inner), dtype=np.float32)
    rc = L.probe_ssm_conv(dev.encode(), case.d_conv, case.d_inner, case.n_t, case.n_s, case.view_sx, case.view_c, ptrs([sx.parent, c.parent]), out.ctypes.data)
    return result(rc, raw, f"probe_ssm_conv({dev}, {case})", out)


def ssm_scan(dev: str, case: ScanCase, views=None, raw: bool = False):
    """SSM_SCAN of `case` on `dev`: (y f32 [n_s, n_t, d_inner], final states f32 [n_s, d_inner, d_state])"""
    L = _lib()
    v = views or case.views()
    parents = [w.parent for w in v[:4]] + ([v[4].parent, v[5].parent] if case.bc_rank < 0 else [v[4].parent])
    out = np.zeros(case.n_y + case.d_state * case.d_inner * case.n_s, dtype=np.float32)
    rc = L.probe_ssm_scan(dev.encode(), case.d_state, case.d_inner, case.n_t, case.n_s, case.bc_rank, ptrs(parents), out.ctypes.data)
    return result(rc, raw, f"probe_ssm_scan({dev}, {case})",
                   (out[: case.n_y].reshape(case.n_s, case.n_t, case.d_inner), out[case.n_y:].reshape(case.n_s, case.d_inner, case.d_state)))


def ulps_apart(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """distance in f32 ulps (0 for bit-identical values; +0 and -0 are 0 apart)"""
    def ordered(x):
        i = np.ascontiguousarray(x, dtype=np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))
