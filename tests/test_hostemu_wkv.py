"""CPU-only: the per-element math of RWKV_WKV6 and GATED_LINEAR_ATTN (ggml_b200/csrc/b200_wkv.cuh) compiled for the HOST through
tests/hostemu/shim (tests/hostemu/wkv_emu.cpp walks sequences, heads, tokens and columns as ops.cu's wkv_kernel does) and checked against
the reference's own ggml-cpu ops, one-node graphs through oracle/wkv_probe.cpp.

  * Head sizes that are a multiple of every CPU build's vector width (8 with AVX2, 16 with AVX-512) run ggml-cpu's fused vector path in
    every column: there the host-compiled code must be BIT-IDENTICAL, which pins the summation order over i and the rounding of every
    multiply and FMA that the device repeats.  Grid: S 16 / 64 / 128, H 1 / 3 / 32, tokens per sequence 1 / 5 / 33, sequences 1 / 3,
    decays exp(-exp(w)) over the trained range, GLA scale 1 and 64^-0.5.
  * Other head sizes (S 8 / 24): ggml-cpu computes its tail columns unfused (the reference is built -std=c11, so gcc does not contract
    there); the result must agree to NMSE 1e-12, and the columns ggml-cpu ran fused must still be bit-identical.
  * The acceptance rules check_rwkv_wkv6 / check_gated_linear_attn (b200_op_checks.h), which the launchers and supports_op share: the
    codes are pinned, and the WKV6 / GLA nodes of the rwkv6 and qrwkv presets of oracle/rwkv_graph.cpp are accepted."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import ggml_b200 as g
from oracle import oracle as O
from oracle import wkv as W

ROOT = Path(__file__).resolve().parents[1]
EMU = ROOT / "tests" / "hostemu"
OK, EUNSUPPORTED, EINVAL = 0, -1, -2


@pytest.fixture(scope="module")
def emu():
    out = EMU / "_build"
    out.mkdir(exist_ok=True)
    so = out / "libwkv_emu.so"
    srcs = [EMU / "wkv_emu.cpp", EMU / "shim" / "cuda_shim.h", ROOT / "ggml_b200" / "csrc" / "b200_wkv.cuh",
            ROOT / "ggml_b200" / "csrc" / "b200_op_checks.h", ROOT / "include" / "ggml-b200.h"]
    if not so.exists() or so.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", "-Werror",
               f"-I{EMU / 'shim'}", "-o", str(so), str(EMU / "wkv_emu.cpp")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(str(so))
    L.emu_rwkv_wkv6.restype = None
    L.emu_rwkv_wkv6.argtypes = [C.c_void_p] * 7 + [C.c_int64] * 4
    L.emu_gated_linear_attn.restype = None
    L.emu_gated_linear_attn.argtypes = [C.c_void_p] * 6 + [C.c_int64] * 4 + [C.c_float]
    L.emu_check_rwkv_wkv6.argtypes = [C.POINTER(g.TensorDesc)] * 7
    L.emu_check_gated_linear_attn.argtypes = [C.POINTER(g.TensorDesc)] * 6
    return L


def emu_wkv(L, case: W.WkvCase, srcs):
    out = np.zeros((case.T + case.S * case.n_seqs) * case.S * case.H, dtype=np.float32)
    p = [a.ctypes.data for a in srcs] + [out.ctypes.data]
    if case.gla:
        L.emu_gated_linear_attn(*p, case.S, case.H, case.T, case.n_seqs, case.scale)
    else:
        L.emu_rwkv_wkv6(*p, case.S, case.H, case.T, case.n_seqs)
    return case.split(out)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def ulps(a, b):
    def ordered(x):
        i = np.ascontiguousarray(x, dtype=np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return int(np.abs(ordered(a) - ordered(b)).max())


CASES = W.grid(False) + W.grid(True)
TAILS = W.tail_grid(False) + W.tail_grid(True)


def test_wkv_grid_covers_the_axes():
    for gla in (False, True):
        cs = [c for c in CASES if c.gla == gla]
        assert {c.S for c in cs} == set(W.GRID_S) and {c.H for c in cs} == set(W.GRID_H)
        assert {c.n_seq_tok for c in cs} == set(W.GRID_TOK) and {c.n_seqs for c in cs} == set(W.GRID_SEQS)
        assert all(c.S % 16 == 0 for c in cs)
    assert {c.scale for c in CASES if c.gla} == set(W.GLA_SCALES)
    assert {c.S for c in TAILS} == set(W.TAIL_S) and all(c.S % 8 or c.S % 16 for c in TAILS)
    decay = np.concatenate([c.sources()[4 if not c.gla else 3].ravel() for c in CASES[:6]])
    assert decay.min() < 1e-3 and decay.max() > 0.999 and ((decay > 0.3) & (decay < 0.7)).any()


@pytest.mark.parametrize("case", CASES, ids=[str(c).replace(" ", "-") for c in CASES])
def test_host_compiled_wkv_is_bit_identical_to_ggml_cpu(case, emu, ref):
    srcs = case.sources()
    y, st = emu_wkv(emu, case, srcs)
    wy, wst = W.wkv("CPU", case, srcs)
    assert np.isfinite(wy).all() and np.isfinite(wst).all(), str(case)
    assert np.array_equal(bits(y), bits(wy)), (str(case), "y", ulps(y, wy))
    assert np.array_equal(bits(st), bits(wst)), (str(case), "states", ulps(st, wst))


@pytest.mark.parametrize("case", TAILS, ids=[str(c).replace(" ", "-") for c in TAILS])
def test_host_compiled_wkv_tail_head_sizes(case, emu, ref):
    srcs = case.sources()
    y, st = emu_wkv(emu, case, srcs)
    wy, wst = W.wkv("CPU", case, srcs)
    assert O.nmse(y, wy) <= 1e-12 and O.nmse(st, wst) <= 1e-12, (str(case), O.nmse(y, wy), O.nmse(st, wst))
    fused = (case.S // W.cpu_vector_width()) * W.cpu_vector_width()       # the columns ggml-cpu ran through its vector path
    assert np.array_equal(bits(y[..., :fused]), bits(wy[..., :fused])), str(case)
    assert np.array_equal(bits(st[..., :fused]), bits(wst[..., :fused])), str(case)


# ------------------------------------------------------------------ the acceptance rules
def wkv_descs(S, H, T, n_seqs, dst_tokens=None):
    """k, v, a, b [S, H, T], tf [S, H], state [S S H, n_seqs] and dst [S H, T + S n_seqs] of zero host tensors (torch order reversed)"""
    z = lambda *shape: torch.zeros(shape)
    src = [g.strided_desc(z(T, H, S)) for _ in range(4)]
    tf = g.strided_desc(z(H, S))
    s = g.strided_desc(z(n_seqs, S * S * H))
    d = g.strided_desc(z((T if dst_tokens is None else dst_tokens) + S * n_seqs, S * H))
    return src, tf, s, d


def codes(L, src, tf, s, d):
    """(WKV6, GLA) verdicts of one set of descriptors"""
    k, v, a, b = src
    return (L.emu_check_rwkv_wkv6(C.byref(k), C.byref(v), C.byref(a), C.byref(tf), C.byref(b), C.byref(s), C.byref(d)),
            L.emu_check_gated_linear_attn(C.byref(k), C.byref(v), C.byref(a), C.byref(b), C.byref(s), C.byref(d)))


def test_wkv_check_codes(emu):
    L = emu
    assert codes(L, *wkv_descs(64, 32, 1, 1)) == (OK, OK)
    assert codes(L, *wkv_descs(64, 32, 0, 2)) == (OK, OK)                       # T = 0: nothing to do, as on the CPU
    assert codes(L, *wkv_descs(256, 2, 3, 1)) == (OK, OK)                       # the head-size limit
    assert codes(L, *wkv_descs(257, 1, 3, 1)) == (EUNSUPPORTED, EUNSUPPORTED)
    assert codes(L, *wkv_descs(64, 4, 5, 2)) == (EINVAL, EINVAL)                # T % n_seqs != 0
    assert codes(L, *wkv_descs(8, 1, 0, 0)) == (OK, OK)
    assert codes(L, *wkv_descs(8, 1, 2, 0)) == (EINVAL, EINVAL)                 # tokens without a sequence
    assert codes(L, *wkv_descs(1, 65536, 1, 1)) == (EUNSUPPORTED, EUNSUPPORTED)  # grid limits
    assert codes(L, *wkv_descs(1, 1, 65536, 65536)) == (EUNSUPPORTED, EUNSUPPORTED)
    assert codes(L, *wkv_descs(1, 1, 65535, 65535)) == (OK, OK)
    assert codes(L, *wkv_descs(16, 2, 3, 1, dst_tokens=4)) == (EUNSUPPORTED, EUNSUPPORTED)   # dst extent
    src, tf, s, d = wkv_descs(16, 2, 3, 1)
    half = g.strided_desc(torch.zeros(3, 2, 16, dtype=torch.float16))
    assert codes(L, [src[0], src[1], half, src[3]], tf, s, d) == (EUNSUPPORTED, EUNSUPPORTED)   # f16
    strided = g.strided_desc(torch.zeros(3, 2, 32)[:, :, :16])
    assert codes(L, [src[0], strided, src[2], src[3]], tf, s, d) == (EUNSUPPORTED, EUNSUPPORTED)  # v not packed
    assert codes(L, [src[0], src[1], src[2], strided], tf, s, d) == (EUNSUPPORTED, EUNSUPPORTED)  # td / g not packed
    assert codes(L, [src[0], g.strided_desc(torch.zeros(3, 2, 17)), src[2], src[3]], tf, s, d) == (EUNSUPPORTED, EUNSUPPORTED)
    assert codes(L, src, g.strided_desc(torch.zeros(2, 15)), s, d)[0] == EUNSUPPORTED                # tf size (WKV6 only)
    assert codes(L, src, g.strided_desc(torch.zeros(2, 32)[:, :16]), s, d)[0] == EUNSUPPORTED         # tf not packed
    assert codes(L, src, g.strided_desc(torch.zeros(2 * 16)), s, d)[0] == OK                       # any shape of S H values
    assert codes(L, src, tf, g.strided_desc(torch.zeros(1, 16 * 16 * 2 + 1)), d) == (EUNSUPPORTED, EUNSUPPORTED)   # state size
    assert codes(L, src, tf, g.strided_desc(torch.zeros(16 * 16 * 2, 1)), d) == (EUNSUPPORTED, EUNSUPPORTED)       # n_seqs is ne1


@pytest.mark.parametrize("preset,H,n_seqs", [("rwkv6", 32, 2), ("qrwkv", 32, 1)])
def test_wkv_nodes_of_the_presets_are_accepted(emu, preset, H, n_seqs):
    # oracle/rwkv_graph.cpp: head size 64, a 7-token prompt per sequence, then one token per sequence per decode step
    for n_t in (7, 1):
        c = codes(emu, *wkv_descs(64, H, n_t * n_seqs, n_seqs))
        assert c[1 if preset == "qrwkv" else 0] == OK, (preset, n_t, c)
