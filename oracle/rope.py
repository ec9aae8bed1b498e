"""TEST INFRASTRUCTURE ONLY: GGML_OP_ROPE cases and the reference's ROPE through oracle/_ref/libggml_rope_probe.so (oracle/rope_probe.cpp).

`Case` describes one ROPE node (shape, type, mode, partial rotation, freq factors, YaRN, positions, strided view); `grid()` is the set the
CPU (host-compiled kernel math) and GPU (device kernel) parity tests run; `probe(dev, case)` evaluates a case on a named ggml device
("CPU": ggml-cpu; "B2000": the plug-in, once loaded with oracle.Ref().load_backend)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import oracle as O
from .probe import probe_lib, result

ROPE_NORM, ROPE_NEOX, ROPE_MROPE, ROPE_VISION = 0, 2, 8, 24
MODE_NAMES = {ROPE_NORM: "norm", ROPE_NEOX: "neox", ROPE_MROPE: "mrope", ROPE_VISION: "vision"}


@dataclass
class Case:
    type: int                     # O.F32 / O.F16
    ne: tuple                     # (ne0, n_head, n_pos, ne3)
    n_dims: int
    mode: int
    sections: tuple = (0, 0, 0, 0)
    ff: bool = False
    ext_factor: float = 0.0
    freq_scale: float = 1.0
    attn_factor: float = 1.0
    view: bool = False
    inplace: bool = False
    n_ctx_orig: int = 512
    freq_base: float = 10000.0
    beta_fast: float = 32.0
    beta_slow: float = 1.0
    seed: int = 0
    positions: tuple | None = None  # the positions, cycled over n_pos (every stream in MROPE); None: random in [0, 4096) with 4095 first
    llama3_ff: bool = False         # with ff: llama-3's factors (llama3_freq_factors) instead of uniform(1, 4) noise

    @property
    def multi(self) -> bool:
        return bool(self.mode & ROPE_MROPE)

    @property
    def parent_ne(self) -> tuple:
        ne0, ne1, ne2, ne3 = self.ne
        return (ne0 * 2, ne1 * 4, ne2 * 3, ne3) if self.view else self.ne

    def inputs(self):
        """(x: the parent tensor's elements in ggml order, pos, freq factors or None)"""
        rng = np.random.default_rng(1000 + self.seed)
        n = int(np.prod(self.parent_ne))
        x = rng.uniform(-1, 1, n).astype(np.float32)
        if self.type == O.F16:
            x = x.astype(np.float16)
        pos = rng.integers(0, 4096, self.ne[2] * (4 if self.multi else 1)).astype(np.int32)
        pos[0] = 4095
        if self.positions is not None:
            pos = np.resize(np.array(self.positions, dtype=np.int32), pos.size)
        ff = None
        if self.ff:
            nff = self.n_dims if self.mode == ROPE_VISION else self.n_dims // 2
            if self.llama3_ff:
                ff = llama3_freq_factors(self.n_dims, self.freq_base)
            else:
                ff = rng.uniform(1.0, 4.0, max(nff, 1)).astype(np.float32)
        return x, pos, ff

    def __str__(self):
        ff = "llama3" if self.ff and self.llama3_ff else int(self.ff)
        pos = "" if self.positions is None else f" pos={min(self.positions)}..{max(self.positions)} ({len(self.positions)} cycled)"
        return (f"{O.TYPE_NAMES[self.type]} {MODE_NAMES[self.mode]} ne={self.ne} n_dims={self.n_dims} sec={self.sections} ff={ff} "
                f"ef={self.ext_factor} fs={self.freq_scale} af={self.attn_factor} base={self.freq_base:g} view={int(self.view)} "
                f"inplace={int(self.inplace)}{pos}")


def llama3_freq_factors(n_dims: int, freq_base: float, factor: float = 8.0, low_freq_factor: float = 1.0, high_freq_factor: float = 4.0,
                        n_ctx_orig: int = 8192) -> np.ndarray:
    """the rope_freqs of a llama-3.1 model (its published rope-scaling rule): 1 for pairs whose wavelength is under
    n_ctx_orig / high_freq_factor, `factor` above n_ctx_orig / low_freq_factor, and a smooth ramp between"""
    out = []
    for j in range(n_dims // 2):
        wavelen = 2 * np.pi / freq_base ** (-2.0 * j / n_dims)
        if wavelen < n_ctx_orig / high_freq_factor:
            out.append(1.0)
        elif wavelen > n_ctx_orig / low_freq_factor:
            out.append(factor)
        else:
            smooth = (n_ctx_orig / wavelen - low_freq_factor) / (high_freq_factor - low_freq_factor)
            out.append(1.0 / ((1.0 - smooth) / factor + smooth))
    return np.array(out, dtype=np.float32)


def grid(inplace: bool = False) -> list:
    """4 modes x f32/f16 x (n_dims < ne0, n_dims = ne0) x freq factors off/on x ext_factor 0/0.7465 x freq_scale 1/1.4245, positions up to
    4095; every other case reads its input through a strided view.  VISION fixes n_dims = ne0/2, so its two variants differ in the sections.
    inplace: NORM / NEOX cases in the in-place form (no view) in addition."""
    out = []
    seed = 0
    for mode in (ROPE_NORM, ROPE_NEOX, ROPE_MROPE, ROPE_VISION):
        for t in (O.F32, O.F16):
            for partial in (True, False):
                if mode == ROPE_NORM:
                    ne, nd, sec = (64, 5, 7, 2), (32 if partial else 64), (0, 0, 0, 0)
                elif mode == ROPE_NEOX:
                    ne, nd, sec = (80, 6, 5, 1), (20 if partial else 80), (0, 0, 0, 0)
                elif mode == ROPE_MROPE:
                    ne, nd, sec = (128, 3, 6, 1), (96 if partial else 128), ((10, 8, 6, 4) if partial else (21, 21, 21, 0))
                else:
                    ne, nd, sec = (80, 4, 6, 1), 40, ((10, 10, 0, 0) if partial else (6, 4, 5, 5))
                for ff in (False, True):
                    for ef in (0.0, 0.7465):
                        for fs in (1.0, 1.4245):
                            seed += 1
                            out.append(Case(t, ne, nd, mode, sec, ff, ef, fs, attn_factor=(1.4245 if seed % 3 == 0 else 1.0), view=bool(seed % 2),
                                            n_ctx_orig=(0 if seed % 5 == 0 else 512), seed=seed))
                            if inplace and mode in (ROPE_NORM, ROPE_NEOX) and seed % 4 == 1:
                                out.append(Case(t, ne, nd, mode, sec, ff, ef, fs, inplace=True, seed=seed))
    return out


SIGNATURES = {
    "probe_rope": [C.c_char_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                   C.c_int] + [C.c_float] * 6 + [C.c_void_p],
}


def probe(dev: str, case: Case) -> np.ndarray:
    """ROPE of `case` on ggml device `dev`: the result, contiguous, in ggml order (flat)"""
    L = probe_lib("rope", "make -C oracle -f decoders.mk llama", SIGNATURES)
    x, pos, ff = case.inputs()
    ne = np.array(case.ne, dtype=np.int64)
    sec = np.array(case.sections, dtype=np.int32)
    out = np.empty(int(np.prod(case.ne)), dtype=x.dtype)
    rc = L.probe_rope(dev.encode(), case.type, ne.ctypes.data, int(case.view), int(case.inplace), x.ctypes.data, pos.ctypes.data,
                      ff.ctypes.data if ff is not None else None, 0 if ff is None else ff.size, case.n_dims, case.mode, sec.ctypes.data,
                      case.n_ctx_orig, case.freq_base, case.freq_scale, case.ext_factor, case.attn_factor, case.beta_fast, case.beta_slow,
                      out.ctypes.data)
    return result(rc, False, f"probe_rope({dev}, {case})", out)
