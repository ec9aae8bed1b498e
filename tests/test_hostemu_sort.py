"""CPU-only: the ARGSORT network (ggml_b200/csrc/b200_sort.cuh) compiled for the HOST through tests/hostemu/shim (tests/hostemu/sort_emu.cpp
runs its steps in the order ops.cu's argsort_kernel does) and checked against the reference's own ggml-cpu ARGSORT, one-node graphs through
oracle/moe_probe.cpp.  Row lengths 1 to 1024 (powers of two and not), both orders:
  * tie-free rows: the same indices as ggml-cpu;
  * rows with ties and +-0: the same sequence of values as ggml-cpu, ties in ascending index (ggml-cpu's exchange sort leaves equal values
    in an order of its own; DESIGN.md §3);
  * rows with +-inf and NaNs: a permutation, the numbers in order before every NaN."""
import ctypes as C

import numpy as np
import pytest

from hostemu.emu import load
from oracle import moe as M


@pytest.fixture(scope="module")
def emu():
    L = load("sort_emu")
    L.emu_argsort.restype = C.c_int
    L.emu_argsort.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p]
    return L


def emu_argsort(L, rows: np.ndarray, order: int) -> np.ndarray:
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    out = np.empty(rows.shape, dtype=np.int32)
    assert L.emu_argsort(rows.ctypes.data, rows.shape[1], rows.shape[0], order, out.ctypes.data) == 0
    return out


CASES = M.argsort_grid()


def test_sort_grid_covers_the_axes():
    assert {c.ne[0] for c in CASES} == set(M.ARGSORT_LENGTHS) and {c.kind for c in CASES} == set(M.KINDS)


@pytest.mark.parametrize("order", [M.ASC, M.DESC], ids=["asc", "desc"])
@pytest.mark.parametrize("case", CASES, ids=[f"{c.ne[0]}-{c.kind}" for c in CASES])
def test_host_compiled_argsort_matches_ggml_cpu(case, order, emu, ref):
    rows = case.rows()
    got = emu_argsort(emu, rows, order)
    want = M.argsort("CPU", case, order)
    for r in range(rows.shape[0]):
        M.check_sorted_row(rows[r], got[r], order, want[r])


def test_host_compiled_argsort_edge_rules(emu):
    # -0.0 equals +0.0 and ties come out by index; NaNs of any sign / payload last in both orders
    x = np.array([0.0, -0.0, 1.0, np.nan, -np.inf, -0.0, np.inf, 1.0], dtype=np.float32)
    x.view(np.uint32)[3] = 0xFFC00001
    assert emu_argsort(emu, x[None], M.ASC)[0].tolist() == [4, 0, 1, 5, 2, 7, 6, 3]
    assert emu_argsort(emu, x[None], M.DESC)[0].tolist() == [6, 2, 7, 0, 1, 5, 4, 3]
    # the example of DESIGN.md §3: DESC of [b, b, c] with b < c
    assert emu_argsort(emu, np.array([[1.0, 1.0, 2.0]], dtype=np.float32), M.DESC)[0].tolist() == [2, 0, 1]
    assert emu.emu_argsort(x.ctypes.data, 1025, 0, 0, None) == -1
