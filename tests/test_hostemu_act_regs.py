"""CPU-only: the activation-stationary consume form of the superblock mat-vec (Q4_K / Q5_K, n = 1, K <= 4096: each lane keeps its half
of an activation task in registers, lane pairs combine their integer sums, the two rows of a warp pass are reduced over lanes xor 16,
8, 4, 2 with the rows exchanged at the first step), emulated in one warp on the host (tests/hostemu/areg_emu.cpp) and compared bit for bit
with the task-per-lane consume it replaces."""
import ctypes as C

import numpy as np
import pytest

from hostemu.emu import load
from oracle import oracle as O


@pytest.fixture(scope="module")
def emu():
    L = load("areg_emu")
    L.emu_sb_areg_rows.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _inputs(K, rng):
    x_zero_task = rng.uniform(-1, 1, K).astype(np.float32)
    x_zero_task[:256] = 0.0                                   # an all-zero act-task (scale 0)
    return [rng.uniform(-1, 1, K).astype(np.float32), (rng.standard_normal(K) * 7).astype(np.float32), x_zero_task,
            (np.round(rng.uniform(-127, 127, K)) / 2).astype(np.float32)]


@pytest.mark.parametrize("K", [256, 1024, 4096])
@pytest.mark.parametrize("t", [O.Q4_K, O.Q5_K], ids=["q4_K", "q5_K"])
def test_register_resident_rows_bit_identical_to_task_per_lane(t, K, emu, oracle):
    rng = np.random.default_rng(1300 + 7 * t + K)
    nrows = 7                                                 # odd: the last pass repeats the last row
    W = O.random_blocks(t, nrows * K // 256, rng)
    Wp = np.concatenate([W, np.zeros(64, dtype=np.uint8)])
    for x in _inputs(K, rng):
        rec = np.zeros(K // 256 * emu.emu_sb_rec_bytes() + 64, dtype=np.uint8)
        regs, tasks = np.zeros(nrows, dtype=np.float32), np.zeros(nrows, dtype=np.float32)
        lanes = np.zeros((nrows, 32), dtype=np.float32)
        assert emu.emu_sb_areg_rows(t, _p(Wp), nrows, K, _p(x), _p(rec), _p(regs), _p(lanes), _p(tasks)) == 0
        assert np.array_equal(regs.view(np.uint32), tasks.view(np.uint32)), (regs, tasks)
        # every lane of a row's half-warp holds the row's sum
        assert np.array_equal(lanes[:, :16].view(np.uint32), np.repeat(tasks[:, None], 16, 1).view(np.uint32))
        want = oracle.mul_mat(t, W, x, nrows, 1, K).reshape(-1)
        assert O.nmse(tasks, want) < 1e-10, (O.nmse(tasks, want), tasks, want)


def test_unsupported_shapes_are_refused(emu):
    z = np.zeros(8192, dtype=np.float32)
    buf = np.zeros(1 << 16, dtype=np.uint8)
    out = np.zeros(64, dtype=np.float32)
    assert emu.emu_sb_areg_rows(O.Q4_K, _p(buf), 1, 8192, _p(z), _p(buf), _p(out), _p(out), _p(out)) == -1
    assert emu.emu_sb_areg_rows(O.Q6_K, _p(buf), 1, 256, _p(z), _p(buf), _p(out), _p(out), _p(out)) == -1
