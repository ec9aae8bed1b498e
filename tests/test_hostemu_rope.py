"""CPU-only: the per-pair math of the ROPE kernel (ggml_b200/csrc/b200_rope.cuh) compiled for the HOST through tests/hostemu/shim
(tests/hostemu/rope_emu.cpp drives it the way ops.cu's rope_kernel does) and checked against the reference's own ggml-cpu ROPE, one-node
graphs through oracle/rope_probe.cpp.  Covers the four modes (NORM, NEOX, MROPE, VISION), f32 / f16, partial rotation, freq factors,
YaRN, freq_scale, positions up to 4095, strided views and the in-place form: pair-index, section and tail mistakes show up here without
a device.  The constants are derived by ggml_b200.rope_params, the Python mirror of what the plug-in passes to the kernel."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import ggml_b200 as g
from oracle import oracle as O
from oracle import rope as R

ROOT = Path(__file__).resolve().parents[1]
EMU = ROOT / "tests" / "hostemu"


@pytest.fixture(scope="module")
def emu():
    out = EMU / "_build"
    out.mkdir(exist_ok=True)
    so = out / "librope_emu.so"
    srcs = [EMU / "rope_emu.cpp", EMU / "shim" / "cuda_shim.h", ROOT / "ggml_b200" / "csrc" / "b200_rope.cuh",
            ROOT / "ggml_b200" / "csrc" / "b200_op_checks.h"]
    if not so.exists() or so.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        cmd = ["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-pthread", "-mf16c", "-mavx", "-ffp-contract=off", "-Wno-unused-variable",
               f"-I{EMU / 'shim'}", "-o", str(so), str(EMU / "rope_emu.cpp")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(str(so))
    L.emu_rope.restype = C.c_int
    L.emu_rope.argtypes = [C.c_int] + [C.c_void_p] * 8
    return L


def _strides(ne, es):
    nb = [es]
    for i in range(3):
        nb.append(nb[-1] * ne[i])
    return np.array(nb, dtype=np.uint64)


def emu_rope(L, case):
    x, pos, ff = case.inputs()
    es = x.itemsize
    p = g.rope_params(case.n_dims, case.mode, case.sections, case.n_ctx_orig, case.freq_base, case.freq_scale, case.ext_factor,
                      case.attn_factor, case.beta_fast, case.beta_slow)
    ne = np.array(case.ne, dtype=np.int64)
    snb = _strides(case.parent_ne, es)
    if case.inplace:
        dst, dnb = x, snb
    else:
        dst, dnb = np.zeros(int(np.prod(case.ne)), dtype=x.dtype), _strides(case.ne, es)
    rc = L.emu_rope(0 if case.type == O.F32 else 1, ne.ctypes.data, x.ctypes.data, snb.ctypes.data, dst.ctypes.data, dnb.ctypes.data,
                    pos.ctypes.data, ff.ctypes.data if ff is not None else None, C.addressof(p))
    assert rc == 0
    return dst


CASES = R.grid(inplace=True)


def test_rope_grid_covers_the_axes():
    axes = {(c.mode, c.type, c.n_dims, c.sections, c.ff, c.ext_factor, c.freq_scale) for c in CASES}
    assert len(axes) == 4 * 2 * 2 * 2 * 2 * 2                  # mode x type x (partial / full rotation) x freq factors x YaRN x freq_scale
    assert any(c.view for c in CASES) and any(c.inplace for c in CASES)


@pytest.mark.parametrize("case", CASES, ids=[f"{i}" for i in range(len(CASES))])
def test_host_compiled_rope_matches_ggml_cpu(case, emu, ref):
    want = R.probe("CPU", case).astype(np.float64)
    got = emu_rope(emu, case).astype(np.float64)
    err = O.nmse(got, want)
    assert err <= 1e-12, (str(case), err)
