"""TEST INFRASTRUCTURE ONLY: GGML_OP_RWKV_WKV6 / GGML_OP_GATED_LINEAR_ATTN / GGML_OP_SQR / GGML_OP_SQRT cases and the reference's ops through
oracle/_ref/libggml_wkv_probe.so (oracle/wkv_probe.cpp).

`WkvCase` describes one WKV6 or GLA node (head size S, heads H, tokens per sequence, sequences, GLA scale) and makes its data from a seed;
`grid()` / `tail_grid()` are the sets the CPU (host-compiled b200_wkv.cuh) and GPU (device kernel) parity tests run; `wkv(dev, case)` and
`sqr_sqrt(dev, op, x)` evaluate on a named ggml device ("CPU": ggml-cpu; "B2000": the plug-in, once loaded with oracle.Ref().load_backend).
Arrays are in ggml's order reversed: k, v, r / q, td / g [T, H, S], tf [H, S], the state [n_seqs, H, S, S] (state[i][j] at [q, h, i, j])."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import oracle as O
from .probe import probe_lib, ptrs, result

GLA_SCALES = (1.0, 64 ** -0.5)


@dataclass
class WkvCase:
    S: int
    H: int
    n_seq_tok: int
    n_seqs: int
    gla: bool = False
    scale: float = 1.0          # GLA only
    seed: int = 0

    @property
    def T(self):
        return self.n_seq_tok * self.n_seqs

    def sources(self):
        """WKV6: k, v, r, tf, td, state; GLA: k, v, q, g, state (f32, contiguous)"""
        rng = np.random.default_rng(11000 + self.seed)
        S, H, T = self.S, self.H, self.T
        f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
        k = f(rng.standard_normal((T, H, S)) * 0.5)
        v = f(rng.standard_normal((T, H, S)))
        r = f(rng.standard_normal((T, H, S)))
        # decay / gate exp(-exp(w)), w over the range trained RWKV-6 layers reach: from ~1 (forgets at once) to ~0.9997 (keeps)
        w = f(np.exp(-np.exp(rng.uniform(-8.0, 2.0, (T, H, S)))))
        state = f(rng.standard_normal((self.n_seqs, H, S, S)))
        if self.gla:
            return [k, v, r, w, state]
        tf = f(rng.standard_normal((H, S)) * 0.5)
        return [k, v, r, tf, w, state]

    def split(self, flat: np.ndarray):
        """(y [T, H, S], final states [n_seqs, H, S, S]) of the flat result"""
        n_y = self.T * self.H * self.S
        return flat[:n_y].reshape(self.T, self.H, self.S), flat[n_y:].reshape(self.n_seqs, self.H, self.S, self.S)

    def __str__(self):
        op = f"gla scale={self.scale:.4g}" if self.gla else "wkv6"
        return f"{op} S={self.S} H={self.H} n_seq_tok={self.n_seq_tok} n_seqs={self.n_seqs}"


GRID_S, GRID_H, GRID_TOK, GRID_SEQS = (16, 64, 128), (1, 3, 32), (1, 5, 33), (1, 3)
TAIL_S = (8, 24)


def grid(gla: bool) -> list:
    """S x H x tokens per sequence x sequences; GLA alternates its scale between 1 and 64^-0.5"""
    out, i = [], 0
    for S in GRID_S:
        for H in GRID_H:
            for nt in GRID_TOK:
                for ns in GRID_SEQS:
                    out.append(WkvCase(S, H, nt, ns, gla, GLA_SCALES[i % 2] if gla else 1.0, seed=i))
                    i += 1
    return out


def tail_grid(gla: bool) -> list:
    """head sizes that are not a multiple of the CPU's vector width (8 with AVX2, 16 with AVX-512) on every build"""
    return [WkvCase(S, H, nt, ns, gla, GLA_SCALES[1] if gla else 1.0, seed=100 + i)
            for i, (S, H, nt, ns) in enumerate((S, H, nt, ns) for S in TAIL_S for H in (1, 3) for nt, ns in ((1, 1), (5, 3)))]


def cpu_vector_width() -> int:
    """columns per vector in the loaded ggml-cpu's WKV6 / GLA loops: 16 for an AVX-512 build, else 8 (x86-64-v3)"""
    ref = O.Ref()
    req = O.REF_DIR / "native" / "REQUIRED_FLAGS"
    return 16 if ref.native and req.exists() and "__AVX512F__" in req.read_text().split() else 8


# ------------------------------------------------------------------ the probe
SIGNATURES = {
    "probe_rwkv_wkv6": [C.c_char_p] + [C.c_int64] * 4 + [C.c_void_p, C.c_void_p],
    "probe_gated_linear_attn": [C.c_char_p] + [C.c_int64] * 4 + [C.c_float, C.c_void_p, C.c_void_p],
    "probe_sqr_sqrt": [C.c_char_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p],
}


def _lib():
    return probe_lib("wkv", "make -C oracle -f decoders.mk rwkv", SIGNATURES)


def wkv(dev: str, case: WkvCase, srcs=None, raw: bool = False, T: int | None = None):
    """the node of `case` on `dev`: (y, final states), or the probe's code when raw.  T overrides the token count (raw only: a T that
    is not a multiple of n_seqs, which ggml-cpu cannot run)"""
    L = _lib()
    srcs = srcs if srcs is not None else case.sources()
    T = case.T if T is None else T
    out = np.zeros((T + case.S * case.n_seqs) * case.S * case.H, dtype=np.float32)
    if T != case.T:
        assert raw
        srcs = [np.zeros(max(1, T * case.H * case.S), np.float32) if a.shape[0] == case.T and a.ndim == 3 else a for a in srcs]
    if case.gla:
        rc = L.probe_gated_linear_attn(dev.encode(), case.S, case.H, T, case.n_seqs, case.scale, ptrs(srcs), out.ctypes.data)
    else:
        rc = L.probe_rwkv_wkv6(dev.encode(), case.S, case.H, T, case.n_seqs, ptrs(srcs), out.ctypes.data)
    return rc if raw else case.split(result(rc, raw, f"probe({dev}, {case})", out))


def sqr_sqrt(dev: str, op: int, x: np.ndarray, raw: bool = False):
    """SQR (op 0) or SQRT (op 1) of the f32 vector x on `dev`"""
    L = _lib()
    x = np.ascontiguousarray(x, dtype=np.float32)
    out = np.zeros_like(x)
    rc = L.probe_sqr_sqrt(dev.encode(), op, x.size, ptrs([x]), out.ctypes.data)
    return result(rc, raw, f"probe_sqr_sqrt({dev}, {op})", out)
