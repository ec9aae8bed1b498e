"""CPU-only: the per-thread decode logic of the CUDA kernels (format traits, 64-weight unit dot products, element decoders of
ggml_b200/csrc/b200_quants.cuh / b200_dequant.cuh) compiled for the HOST through tests/hostemu/shim and checked against the oracle.
Catches indexing / bit-twiddling mistakes in a block format without a GPU; the `-m gpu` parity tests remain the gate for the
kernels themselves (scheduling, memory movement, PTX-level instructions)."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import oracle as O

ROOT = Path(__file__).resolve().parents[1]
EMU = ROOT / "tests" / "hostemu"


@pytest.fixture(scope="module")
def emu():
    out = EMU / "_build"
    out.mkdir(exist_ok=True)
    so = out / "libhostemu.so"
    srcs = [EMU / "hostemu.cpp", EMU / "shim" / "cuda_shim.h"] + [ROOT / "ggml_b200" / "csrc" / f for f in ("b200_quants.cuh", "b200_dequant.cuh", "b200_sb_tasks.cuh", "b200_tc_dequant.cuh", "b200_iq.cuh", "b200_sb_mma.cuh", "generated/iq_grids.h")]
    if not so.exists() or so.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        cmd = ["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-pthread", "-mf16c", "-mavx", "-ffp-contract=off", "-Wno-unused-variable", "-Wno-unknown-pragmas",
               f"-I{EMU / 'shim'}", "-o", str(so), str(EMU / "hostemu.cpp")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(str(so))
    L.emu_row_dot.restype = C.c_float
    L.emu_row_dot.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    L.emu_dequant.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
    L.emu_act_layout.argtypes = [C.c_int64, C.c_int, C.c_void_p]
    L.emu_row_bytes.restype = C.c_int64
    L.emu_row_bytes.argtypes = [C.c_int, C.c_int64]
    L.emu_tc_dequant_row.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    L.emu_quantize_record.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    L.emu_sb_quantize.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int]
    L.emu_sb_geometry.argtypes = [C.c_int, C.c_void_p]
    L.emu_sb_row_dot.restype = C.c_float
    L.emu_sb_row_dot.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    L.emu_sb_two_row_dot.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    L.emu_sb_row_dot_nc.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.emu_mma_tile.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def supported(emu, t):
    return emu.emu_row_bytes(t, 256) > 0


def act_record(emu, oracle, t, x):
    """the device-side activation record (q | bs | d [| s]) built from the ORACLE's quantized activations"""
    K = x.size
    kq = bool(emu.emu_type_is_kquant(t))
    lay = np.zeros(4, dtype=np.int32)
    emu.emu_act_layout(K, int(kq), _p(lay))
    off_bs, off_d, off_s, nbytes = (int(v) for v in lay)
    rec = np.zeros(nbytes + 64, dtype=np.uint8)
    vdt = oracle.vec_dot_type(t)
    yq = oracle.quantize(vdt, x, simd_q8_0=(vdt == O.Q8_0))
    if vdt == O.Q8_K:
        b = yq.reshape(-1, 292)
        q = b[:, 4:260].reshape(-1).view(np.int8)
        d = b[:, :4].copy().view(np.float32).reshape(-1)
    else:
        bs_ = 34 if vdt == O.Q8_0 else 36
        b = yq.reshape(-1, bs_)
        q = b[:, bs_ - 32:].reshape(-1).view(np.int8)
        d = b[:, :2].copy().view(np.float16).astype(np.float32).reshape(-1)
        if vdt == O.Q8_1:
            assert off_s >= 0, "the record needs the Q8_1 's' section for formats with a minimum"
        if off_s >= 0:                                        # the device quantizer fills 's' for the whole Q8_0 family (same codes and d as Q8_0)
            b1 = oracle.quantize(O.Q8_1, x).reshape(-1, 36)
            assert np.array_equal(b1[:, 4:].reshape(-1).view(np.int8), q)
            s = b1[:, 2:4].copy().view(np.float16).astype(np.float32).reshape(-1)
            rec[off_s:off_s + 4 * s.size] = s.view(np.uint8)
    rec[:K] = q.view(np.uint8)
    bsum = q.reshape(-1, 16).astype(np.int32).sum(1).astype(np.int16)
    rec[off_bs:off_bs + 2 * bsum.size] = bsum.view(np.uint8)
    rec[off_d:off_d + 4 * d.size] = d.view(np.uint8)
    return rec, yq


ALL = list(O.HOT_TYPES) + list(O.NEXT_TYPES) + list(O.IQ_TYPES)


@pytest.mark.parametrize("t", ALL, ids=[O.TYPE_NAMES[t] for t in ALL])
def test_element_decoders_bit_exact(t, emu, oracle):
    if not supported(emu, t):
        pytest.skip("format not implemented in ggml_b200/csrc yet")
    rng = np.random.default_rng(300 + t)
    nb = 512
    blocks = O.random_blocks(t, nb, rng)
    n = nb * oracle.blck_size(t)
    out = np.empty(n, dtype=np.float32)
    assert emu.emu_dequant(t, _p(blocks), _p(out), n) == 0
    assert np.array_equal(out.view(np.uint32), oracle.dequantize(t, blocks, n).view(np.uint32))
    z = np.load(ROOT / "tests" / "golden" / f"quant_{O.TYPE_NAMES[t]}.npz")          # the reference's own blocks
    out = np.empty(z["x"].size, dtype=np.float32)
    assert emu.emu_dequant(t, _p(np.ascontiguousarray(z["blocks"])), _p(out), out.size) == 0
    assert np.array_equal(out.view(np.uint32), z["deq"].view(np.uint32))


@pytest.mark.parametrize("t", ALL, ids=[O.TYPE_NAMES[t] for t in ALL])
def test_unit_dot_products_match_oracle(t, emu, oracle):
    if not supported(emu, t):
        pytest.skip("format not implemented in ggml_b200/csrc yet")
    rng = np.random.default_rng(400 + t)
    for K in (256, 1024, 4096) + ((32, 96, 160) if oracle.blck_size(t) == 32 else ()):          # odd block counts: trailing-block path
        x = rng.uniform(-1, 1, K).astype(np.float32)
        rec, yq = act_record(emu, oracle, t, x)
        for trial in range(6):
            w = O.random_blocks(t, K // oracle.blck_size(t), rng)
            w = np.concatenate([w, np.zeros(64, dtype=np.uint8)])                      # the kernels read aligned words past 2-byte-aligned rows
            got = float(emu.emu_row_dot(t, _p(w), K, _p(rec)))
            want = oracle.vec_dot(t, K, w[:-64], yq)
            scale = float(np.linalg.norm(oracle.dequantize(t, w[:-64], K)) * np.linalg.norm(x)) + 1e-30
            assert abs(got - want) <= 2e-6 * scale, (K, trial, got, want)


def sb_record(emu, oracle, t, x):
    """the superblock kernel's per-act-task activation records (q | s32 | s16 | h32 | d) built from the ORACLE's quantized activations"""
    geo = np.zeros(7, dtype=np.int32)
    assert emu.emu_sb_geometry(t, _p(geo)) == 0
    _, _, REC, OFF_S32, OFF_S16, OFF_H32, OFF_D = (int(v) for v in geo)
    K = x.size
    ntask = K // 256
    vdt = oracle.vec_dot_type(t)
    yq = oracle.quantize(vdt, x, simd_q8_0=(vdt == O.Q8_0))
    if vdt == O.Q8_K:
        b = yq.reshape(-1, 292)
        q = b[:, 4:260].copy().view(np.int8).reshape(ntask, 256)
        d = b[:, :4].copy().view(np.float32).reshape(ntask, 1)
    else:
        hb = 2 if vdt == O.Q8_0 else 4                        # Q8_0: d | 32 codes;  Q8_1: d | s | 32 codes
        b = yq.reshape(-1, 32 + hb)
        q = b[:, hb:].copy().view(np.int8).reshape(ntask, 256)
        d = b[:, :2].copy().view(np.float16).astype(np.float32).reshape(ntask, 8)
        s_half = b[:, 2:4].copy().reshape(ntask, 16) if vdt == O.Q8_1 else None
    rec = np.zeros(ntask * REC + 64, dtype=np.uint8)
    for tt in range(ntask):
        base = tt * REC
        rec[base:base + 256] = q[tt].view(np.uint8)
        s32 = q[tt].reshape(8, 32).astype(np.int32).sum(1).astype(np.int32)
        s16 = q[tt].reshape(16, 16).astype(np.int32).sum(1).astype(np.int16)
        rec[base + OFF_S32:base + OFF_S32 + 32] = s32.view(np.uint8)
        rec[base + OFF_S16:base + OFF_S16 + 32] = s16.view(np.uint8)
        rec[base + OFF_H32:base + OFF_H32 + 16] = s32.astype(np.int16).view(np.uint8)
        if vdt == O.Q8_1:                                     # formats with a minimum: the H32 slot carries the eight fp16 s values
            rec[base + OFF_H32:base + OFF_H32 + 16] = s_half[tt]
        dd = d[tt].astype(np.float32)
        rec[base + OFF_D:base + OFF_D + 4 * dd.size] = dd.view(np.uint8)
    return rec, yq, ntask * REC


HOT = list(O.HOT_TYPES) + [O.Q5_0, O.Q2_K, O.Q3_K, O.Q4_1, O.Q5_1, O.IQ4_NL, O.IQ4_XS]      # + the next formats whose fast-path task dot products are written (not yet dispatched)


@pytest.mark.parametrize("t", HOT, ids=[O.TYPE_NAMES[t] for t in HOT])
def test_superblock_task_dot_products_match_oracle(t, emu, oracle):
    """mmvq_sb.cu's per-lane task dot products (packed 6-bit scale decode, dp2a mins, in-place high nibbles, 2-byte-aligned Q6_K
    words, ...) and their multi-column form: against the oracle, and column by column bit-identical to the single-column form"""
    rng = np.random.default_rng(500 + t)
    for K in (256, 768, 4096):
        xs = [rng.uniform(-1, 1, K).astype(np.float32) for _ in range(5)]
        recs = [sb_record(emu, oracle, t, x) for x in xs]
        stride = recs[0][2]
        allrec = np.concatenate([r[0][:stride] for r in recs] + [np.zeros(64, dtype=np.uint8)])
        for trial in range(4):
            w = O.random_blocks(t, K // oracle.blck_size(t), rng)
            wp = np.concatenate([w, np.zeros(64, dtype=np.uint8)])
            singles = []
            for (rec, yq, _), x in zip(recs, xs):
                got = float(emu.emu_sb_row_dot(t, _p(wp), K, _p(rec)))
                want = oracle.vec_dot(t, K, w, yq)
                scale = float(np.linalg.norm(oracle.dequantize(t, w, K)) * np.linalg.norm(x)) + 1e-30
                assert abs(got - want) <= 2e-6 * scale, (K, trial, got, want)
                singles.append(np.float32(got))
            out = np.zeros(8, dtype=np.float32)
            assert emu.emu_sb_row_dot_nc(t, _p(wp), K, _p(allrec), stride, 5, _p(out)) == 0
            assert np.array_equal(out[:5].view(np.uint32), np.array(singles, dtype=np.float32).view(np.uint32)), (K, trial)
            assert np.all(out[5:] == 0)


@pytest.mark.parametrize("t", [O.Q4_K, O.Q5_K], ids=["q4_K", "q5_K"])
def test_two_row_task_dot_is_bit_identical_to_single_row(t, emu, oracle):
    """the round-2 variant that shares the activation loads between two weight rows (not dispatched yet)"""
    rng = np.random.default_rng(600 + t)
    for K in (256, 4096):
        x = rng.uniform(-1, 1, K).astype(np.float32)
        rec, _, _ = sb_record(emu, oracle, t, x)
        for trial in range(4):
            w0 = np.concatenate([O.random_blocks(t, K // 256, rng), np.zeros(64, dtype=np.uint8)])
            w1 = np.concatenate([O.random_blocks(t, K // 256, rng), np.zeros(64, dtype=np.uint8)])
            out = np.zeros(2, dtype=np.float32)
            assert emu.emu_sb_two_row_dot(t, _p(w0), _p(w1), K, _p(rec), _p(out)) == 0
            want = np.array([emu.emu_sb_row_dot(t, _p(w0), K, _p(rec)), emu.emu_sb_row_dot(t, _p(w1), K, _p(rec))], dtype=np.float32)
            assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), (K, trial)


def _inputs(K):
    rng = np.random.default_rng(700 + K)
    z = np.load(ROOT / "tests" / "golden" / "act_q8.npz")["x"]
    reps = (K + z.size - 1) // z.size
    return [np.tile(z, reps)[:K].astype(np.float32), rng.uniform(-1, 1, K).astype(np.float32), (rng.standard_normal(K) * 7).astype(np.float32),
            np.zeros(K, dtype=np.float32), (np.round(rng.uniform(-127, 127, K)) / 2).astype(np.float32)]


@pytest.mark.parametrize("t", [O.Q4_0, O.Q4_1, O.Q4_K], ids=["q8_0-family", "q8_1-family", "q8_K-family"])
def test_activation_quantizers_in_an_emulated_warp(t, emu, oracle):
    """the device activation quantizers (warp shuffles emulated by 32 host threads in lockstep) are bit-exact against the oracle's
    restatement of the CPU backend's quantizers: both record layouts, including the Q8_1 's' section"""
    kq = bool(emu.emu_type_is_kquant(t))
    for K in (256, 768, 3072) + (() if kq else (32, 96, 160, 288)):          # the Q8_0 family also takes K % 256 != 0
        for x in _inputs(K):
            want_rec, _ = act_record(emu, oracle, t, x)
            got = np.zeros(want_rec.size, dtype=np.uint8)
            n = emu.emu_quantize_record(int(kq), _p(x), K, _p(got))
            if kq:                                            # bsums of all-zero superblocks: the reference leaves them uninitialised, the device writes 0
                pass
            assert np.array_equal(got[:n], want_rec[:n]), (K,)
            if K % 256 == 0:                                  # the superblock-kernel record (whole act-tasks); Q4_1: Q8_1 's' in the H32 slot
                want_sb, _, nb = sb_record(emu, oracle, t, x)
                got_sb = np.zeros(want_sb.size, dtype=np.uint8)
                assert emu.emu_sb_quantize(int(kq), _p(x), K, _p(got_sb), int(t == O.Q4_1)) == nb
                assert np.array_equal(got_sb[:nb], want_sb[:nb]), (K,)


TC_TYPES = [O.Q4_0, O.Q8_0, O.Q4_K, O.Q5_K, O.Q6_K, O.Q4_1, O.Q5_0, O.Q5_1, O.IQ4_NL, O.IQ4_XS, O.Q2_K, O.Q3_K]


@pytest.mark.parametrize("t", TC_TYPES, ids=[O.TYPE_NAMES[t] for t in TC_TYPES])
def test_gemm_operand_dequantization_matches_oracle(t, emu, oracle):
    """the GEMM's packed-half dequantization (b200_tc_dequant.cuh, mmq_tc2.cu; integer code -> 1024 + code by PRMT, HSUB2, HMUL2 / HFMA2): every fp16 weight within
    fp16 rounding of the oracle's exact dequantization (the scale product and the result are each rounded once to fp16)"""
    rng = np.random.default_rng(800 + t)
    K = 1024
    for trial in range(6):
        w = O.random_blocks(t, K // oracle.blck_size(t), rng) if trial % 2 else None
        if w is None:
            z = np.load(ROOT / "tests" / "golden" / f"quant_{O.TYPE_NAMES[t]}.npz")
            w = np.ascontiguousarray(z["blocks"][:oracle.row_size(t, K)])
        wp = np.concatenate([w, np.zeros(64, dtype=np.uint8)])
        out = np.zeros(K, dtype=np.uint16)
        rc = emu.emu_tc_dequant_row(t, _p(wp), K, _p(out))
        if rc != 0:
            pytest.skip("format not in the tensor-core GEMM yet")
        got = out.view(np.float16).astype(np.float32)
        want = oracle.dequantize(t, w, K)
        blk = np.abs(want).reshape(-1, 32).max(1).repeat(32) + 1e-12
        assert np.all(np.abs(got - want) <= 1.5e-3 * blk), (trial, float(np.max(np.abs(got - want) / blk)))


@pytest.mark.parametrize("ncols", [1, 2, 5, 8])
@pytest.mark.parametrize("t", [O.Q4_K, O.Q5_K, O.Q6_K, O.Q4_0, O.Q8_0, O.Q5_0, O.Q4_1, O.Q5_1, O.IQ4_NL, O.IQ4_XS, O.Q2_K, O.Q3_K], ids=lambda t: O.TYPE_NAMES[t])
def test_mma_small_batch_tile_matches_oracle(t, ncols, emu, oracle):
    """b200_sb_mma.cuh (the int8 mma.sync consume path of mmvq_mma.cu) in an emulated warp — fragment loads from the packed rows at a
    padded pitch, the m16n8k32 fragment layout, scale / min application, the planar activation records of the kernel's own quantizer —
    against the oracle's mul_mat (same integer dots, f32 order differs)."""
    rng = np.random.default_rng(1000 * t + ncols)
    K = 1024
    rb = oracle.row_size(t, K)
    W = O.random_blocks(t, 16 * K // oracle.blck_size(t), rng)
    pitch = rb + (16 if t in (O.Q6_K, O.Q2_K, O.Q3_K) else 32)
    rows = np.zeros(16 * pitch + 64, dtype=np.uint8)
    base = (-rows.ctypes.data) % 32                      # 32-byte aligned tile, as a shared-memory stage
    for r in range(16):
        rows[base + r * pitch: base + r * pitch + rb] = W[r * rb:(r + 1) * rb]
    X = rng.uniform(-1, 1, ncols * K).astype(np.float32)
    X[3 * 256:4 * 256] = 0.0                             # an all-zero act-task of column 0
    out = np.zeros((16, 8), dtype=np.float32)
    assert emu.emu_mma_tile(t, C.c_void_p(rows.ctypes.data + base), pitch, K, _p(X), ncols, _p(out)) == 0
    want = oracle.mul_mat(t, W, X, 16, ncols, K)          # [ncols, 16]
    got = out[:, :ncols].T
    assert O.nmse(got, want) < 1e-10, (O.nmse(got, want), got[:, :3], want[:, :3])
