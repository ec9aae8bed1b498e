"""CPU-only: the per-element math of SSM_CONV and SSM_SCAN (ggml_b200/csrc/b200_ssm.cuh) compiled for the HOST through tests/hostemu/shim
(tests/hostemu/ssm_emu.cpp indexes the sources as ops.cu's ssm_conv_kernel / ssm_scan_kernel do) and checked against the reference's own
ggml-cpu ops, one-node graphs through oracle/ssm_probe.cpp.  Compiled for the host, with glibc's expf / log1pf, both must be
BIT-IDENTICAL to ggml-cpu: that pins the order of every sum and the separate rounding of every multiply and add, which the device keeps.
The grid covers d_conv 2 / 4 / 8, n_t 1 / 5 / 64, n_s 1 / 3, d_state 1 / 16 / 64 / 256, dt on both sides of the softplus cut-off at 20,
strided conv inputs and B / C as strided views of one x_db, as in the Mamba layer."""
import ctypes as C

import numpy as np
import pytest

from hostemu.emu import load
from oracle import ssm as S


class EmuTensor(C.Structure):
    _fields_ = [("data", C.c_void_p), ("ne", C.c_int64 * 4), ("nb", C.c_uint64 * 4)]


def emu_tensor(v: S.View) -> EmuTensor:
    t = EmuTensor()
    t.data = v.parent.ctypes.data + v.offs
    for i in range(4):
        t.ne[i], t.nb[i] = v.ne[i], v.nb[i]
    return t


@pytest.fixture(scope="module")
def emu():
    L = load("ssm_emu")
    L.emu_ssm_conv.restype = None
    L.emu_ssm_conv.argtypes = [C.POINTER(EmuTensor), C.POINTER(EmuTensor), C.c_void_p, C.c_int64]
    L.emu_ssm_scan.restype = None
    L.emu_ssm_scan.argtypes = [C.POINTER(EmuTensor), C.c_void_p]
    return L


def emu_ssm_conv(L, case: S.ConvCase, views):
    sx, c = (emu_tensor(v) for v in views)
    out = np.zeros((case.n_s, case.n_t, case.d_inner), dtype=np.float32)
    L.emu_ssm_conv(C.byref(sx), C.byref(c), out.ctypes.data, case.n_t)
    return out


def emu_ssm_scan(L, case: S.ScanCase, views):
    ts = (EmuTensor * 6)(*[emu_tensor(v) for v in views])
    out = np.zeros(case.n_y + case.d_state * case.d_inner * case.n_s, dtype=np.float32)
    L.emu_ssm_scan(ts, out.ctypes.data)
    return out[: case.n_y].reshape(case.n_s, case.n_t, case.d_inner), out[case.n_y:].reshape(case.n_s, case.d_inner, case.d_state)


CONV = S.conv_grid()
SCAN = S.scan_grid()


def test_ssm_grids_cover_the_axes():
    assert {c.d_conv for c in CONV} == set(S.CONV_D_CONV) and {c.n_t for c in CONV} == set(S.CONV_N_T) and {c.n_s for c in CONV} == set(S.CONV_N_S)
    assert {(c.view_sx, c.view_c) for c in CONV} == {(0, 0), (3, 3), (3, 0)}
    assert {c.d_state for c in SCAN} == set(S.SCAN_D_STATE) and {c.n_t for c in SCAN} == set(S.SCAN_N_T) and {c.n_s for c in SCAN} == set(S.SCAN_N_S)
    assert {c.bc_rank >= 0 for c in SCAN} == {True, False}
    dt = np.concatenate([S.read(c.views()[2]).ravel() for c in SCAN])
    assert (dt > 20).any() and (dt == 20).any() and ((dt < 20) & (dt > 10)).any() and (dt < 0).any()


def test_views_read_what_the_probe_reads():
    # the numpy model of a transposed / strided source (S.read) against ggml-cpu's CONCAT of it, which copies words bit for bit
    case = S.ConcatCase(S.F32, (3, 5, 2, 1), (4, 5, 2, 1), 0, 1, 2, seed=3)
    pa, pb = case.parents()
    want = np.concatenate([S.read(S.make_view(pa, case.ne_a, 1)), S.read(S.make_view(pb, case.ne_b, 2))], axis=3)
    got = S.concat("CPU", case)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("case", CONV, ids=[f"dc{c.d_conv}-nt{c.n_t}-ns{c.n_s}-v{c.view_sx}{c.view_c}" for c in CONV])
def test_host_compiled_ssm_conv_is_bit_identical_to_ggml_cpu(case, emu, ref):
    views = case.views()
    got = emu_ssm_conv(emu, case, views)
    want = S.ssm_conv("CPU", case, views)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (str(case), int(S.ulps_apart(got, want).max()))


@pytest.mark.parametrize("case", SCAN, ids=[f"ds{c.d_state}-nt{c.n_t}-ns{c.n_s}-bc{c.bc_rank}" for c in SCAN])
def test_host_compiled_ssm_scan_is_bit_identical_to_ggml_cpu(case, emu, ref):
    views = case.views()
    y, st = emu_ssm_scan(emu, case, views)
    wy, wst = S.ssm_scan("CPU", case, views)
    assert np.isfinite(wy).all() and np.isfinite(wst).all(), str(case)
    assert np.array_equal(y.view(np.uint32), wy.view(np.uint32)), (str(case), "y", int(S.ulps_apart(y, wy).max()))
    assert np.array_equal(st.view(np.uint32), wst.view(np.uint32)), (str(case), "states", int(S.ulps_apart(st, wst).max()))
