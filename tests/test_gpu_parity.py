"""GPU parity: the hand-written sm_90a kernels, called through the C ABI (include/ggml-b200.h), against the CPU
oracle on identical seeded inputs and against the reference's golden vectors.

Bars: dequantize / quantize / activation quantizer are BIT-EXACT; MUL_MAT(_ID) within NMSE 1e-10 of the oracle
(f32 summation order is the only difference) — the reference's own gate is 5e-4 (tests/test-backend-ops.cpp:1915)."""
from pathlib import Path

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu

G = Path(__file__).resolve().parent / "golden"
TYPES = list(O.HOT_TYPES)
IDS = [O.TYPE_NAMES[t] for t in TYPES]
TOL = 1e-10


@pytest.fixture(scope="module")
def g():
    import torch
    assert torch.cuda.is_available(), "these tests need an H100"
    import ggml_b200
    ggml_b200.lib()
    return ggml_b200


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def weights(oracle, t, M, K, seed, rng_blocks=False):
    """packed weights: quantized by the oracle for Q4_0/Q8_0; arbitrary valid blocks for K-quants
    (their host-side quantizers are not on the device path) unless golden data is used."""
    rng = np.random.default_rng(seed)
    if t in (O.Q4_0, O.Q8_0) and not rng_blocks:
        w = rng.uniform(-1, 1, M * K).astype(np.float32)
        return np.concatenate([oracle.quantize(t, w[i * K:(i + 1) * K]) for i in range(M)])
    return O.random_blocks(t, M * K // oracle.blck_size(t), rng)


@pytest.mark.parametrize("t", TYPES, ids=IDS)
def test_dequantize_bit_exact(t, g, oracle):
    import torch
    z = np.load(G / f"quant_{O.TYPE_NAMES[t]}.npz")
    for blocks, want in ((z["blocks"], z["deq"]), (z["rnd_blocks"], z["rnd_deq"])):
        got = g.dequantize(t, dev(blocks), want.size).cpu().numpy()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        got16 = g.dequantize(t, dev(blocks), want.size, dtype=torch.float16).cpu().numpy()
        assert np.array_equal(got16.view(np.uint16), want.astype(np.float16).view(np.uint16))
    rng = np.random.default_rng(t)
    nb = 100_000 if t in (O.Q4_0, O.Q8_0) else 20_000
    blocks = O.random_blocks(t, nb, rng)
    n = nb * oracle.blck_size(t)
    assert np.array_equal(g.dequantize(t, dev(blocks), n).cpu().numpy().view(np.uint32), oracle.dequantize(t, blocks, n).view(np.uint32))


@pytest.mark.parametrize("t", [O.Q8_0, O.Q4_0], ids=["q8_0", "q4_0"])
def test_quantize_bit_exact(t, g, oracle):
    z = np.load(G / "act_q8.npz")
    assert np.array_equal(g.quantize(t, dev(z["x"])).cpu().numpy(), z["q8_0_ref" if t == O.Q8_0 else "q4_0_ref"])
    rng = np.random.default_rng(3)
    x = np.concatenate([rng.uniform(-1, 1, 1 << 16), rng.standard_normal(1 << 16) * 50, np.round(rng.uniform(-16, 16, 1 << 14) * 2) / 2]).astype(np.float32)
    assert np.array_equal(g.quantize(t, dev(x)).cpu().numpy(), oracle.quantize(t, x))
    # round trip: dequantize(quantize(x)) on the device == the oracle's
    q = g.quantize(t, dev(x))
    assert np.array_equal(g.dequantize(t, q, x.size).cpu().numpy().view(np.uint32), oracle.dequantize(t, oracle.quantize(t, x), x.size).view(np.uint32))


def unpack_records(rec, K, kq):
    bs_off = (K + 15) & ~15
    d_off = bs_off + ((K // 16 * 2 + 15) & ~15)
    q = rec[:, :K].view(np.int8)
    bs = rec[:, bs_off:bs_off + K // 16 * 2].copy().view(np.int16)
    nd = K // 256 if kq else K // 32
    d = rec[:, d_off:d_off + nd * 4].copy().view(np.float32)
    return q, bs, d


@pytest.mark.parametrize("wt", [O.Q4_0, O.Q4_K], ids=["q8_0-family", "q8_K-family"])
def test_activation_quantizer_bit_exact(wt, g, oracle):
    z = np.load(G / "act_q8.npz")
    rng = np.random.default_rng(8)
    K = 3072
    X = np.stack([z["x"][:K], rng.uniform(-1, 1, K), rng.standard_normal(K) * 7, np.zeros(K), np.round(rng.uniform(-127, 127, K)) / 2]).astype(np.float32)
    rec = g.quantize_activations(wt, dev(X)).cpu().numpy()
    kq = wt == O.Q4_K
    q, bs, d = unpack_records(rec, K, kq)
    for r in range(X.shape[0]):
        if kq:
            want = oracle.quantize(O.Q8_K, X[r]).reshape(-1, 292)
            assert np.array_equal(q[r], want[:, 4:260].reshape(-1).view(np.int8))
            assert np.array_equal(d[r].view(np.uint32), want[:, :4].copy().view(np.uint32).reshape(-1))
            nz = ~np.all(want[:, 4:260] == 0, axis=1)
            assert np.array_equal(bs[r].reshape(-1, 16)[nz], want[:, 260:].copy().view(np.int16).reshape(-1, 16)[nz])
        else:
            want = oracle.quantize(O.Q8_0, X[r], simd_q8_0=True).reshape(-1, 34)
            assert np.array_equal(q[r], want[:, 2:].reshape(-1).view(np.int8))
            assert np.array_equal(d[r], want[:, :2].copy().view(np.float16).astype(np.float32).reshape(-1))
            assert np.array_equal(bs[r], q[r].reshape(-1, 16).astype(np.int32).sum(1).astype(np.int16))


@pytest.mark.parametrize("t", TYPES, ids=IDS)
def test_mul_mat_golden(t, g):
    z = np.load(G / f"mulmat_{O.TYPE_NAMES[t]}.npz")
    for ci in range(int(z["ncases"])):
        M, N, K = (int(v) for v in z[f"shape{ci}"])
        for flags in (g.MM_AUTO, g.MM_GENERIC):
            Y = g.mul_mat(t, dev(z[f"W{ci}"]), dev(z[f"X{ci}"]), M, N, K, flags=flags).cpu().numpy()[0, 0]
            # the tensor-core path (n >= 9) computes with fp16 operands: stated tolerance 1e-4 (reference gate 5e-4); int8 paths 1e-10
            tol = 1e-4 if g.mul_mat_plan(t, M, N, K, flags) == g.MM_GEMM else TOL
            assert O.nmse(Y, z[f"Y{ci}"]) < tol, (ci, M, N, K, flags)


@pytest.mark.parametrize("t", TYPES, ids=IDS)
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 8])
def test_gemv_vs_oracle(t, n, g, oracle):
    # shapes chosen to hit: K-parts 1..8, partial last stage, tiny M, rows-per-stage granules
    for (M, K) in [(1000, 4096), (257, 1024), (64, 11008 // 256 * 256), (24, 256), (4096, 768 if t in (O.Q4_0, O.Q8_0) else 2048), (3000, 2048), (136, 8192)]:
        if g.mul_mat_plan(t, M, n, K, g.MM_GEMV) != g.MM_GEMV:
            continue
        W = weights(oracle, t, M, K, seed=M + K + t)
        X = np.random.default_rng(5678).uniform(-1, 1, n * K).astype(np.float32)
        want = oracle.mul_mat(t, W, X, M, n, K)
        # n = 1 has two kernels: the one-lane-per-256-weights kernel (default) and the 64-weight-unit kernel (V1)
        # (+ its two operating points: dependent launch = 8-warp CTAs + L2 prefetch of static weights; independent launch = 4-warp CTAs)
        for flags in ((g.MM_GEMV, g.MM_GEMV | g.MM_GEMV_V1, g.MM_GEMV | g.MM_SRC0_STATIC, g.MM_GEMV | g.MM_SRC0_STATIC | g.MM_SRC1_STATIC) if n == 1 else (g.MM_GEMV,)):
            if g.mul_mat_plan(t, M, n, K, flags) != g.MM_GEMV:
                continue
            Y = g.mul_mat(t, dev(W), dev(X), M, n, K, flags=flags).cpu().numpy()[0, 0]
            assert O.nmse(Y, want) < TOL, (M, K, n, flags)
            assert np.isfinite(Y).all()


@pytest.mark.parametrize("t", TYPES, ids=IDS)
def test_small_batch_columns_match_single_column(t, g, oracle):
    """2 <= n <= 8 on the dp4a superblock kernel (GGML_B200_MM_GEMV_DP4A) decodes the weights once per task: every column must be
    bit-identical to the n = 1 product with that column (same integer dots, same f32 operations in the same order)."""
    M, K = 1536, 4096
    W = dev(weights(oracle, t, M, K, seed=99))
    rng = np.random.default_rng(7)
    F = g.MM_GEMV | g.MM_GEMV_DP4A
    for n in (2, 3, 4, 7, 8):
        if g.mul_mat_plan(t, M, n, K, F) != g.MM_GEMV:
            continue
        X = rng.uniform(-1, 1, (n, K)).astype(np.float32)
        Y = g.mul_mat(t, W, dev(X), M, n, K, flags=F).cpu().numpy()[0, 0]
        for c in range(n):
            y1 = g.mul_mat(t, W, dev(X[c]), M, 1, K, flags=F).cpu().numpy()[0, 0, 0]
            assert np.array_equal(Y[c], y1), (n, c)


MMA_TYPES = [O.Q4_0, O.Q8_0, O.Q4_K, O.Q5_K, O.Q6_K, O.Q5_0, O.Q4_1, O.Q5_1, O.IQ4_NL, O.IQ4_XS, O.Q2_K, O.Q3_K]


@pytest.mark.parametrize("t", MMA_TYPES, ids=[O.TYPE_NAMES[t] for t in MMA_TYPES])
def test_small_batch_mma_kernel_vs_oracle(t, g, oracle):
    """mmvq_mma.cu (int8 mma.sync consume path, the default for 2 <= n <= 8): against the oracle at whole-row stages (K = 2048, 4096),
    K-sliced stages with a ragged last slice (K = 11008: 43 tasks), ragged M (last tile partly filled), every n in 1..8;
    bitwise repeatable; column c of an n-column launch bit-identical to the kernel's own n = 1 result for that column."""
    rng = np.random.default_rng(17)
    k_sliced = 11008 if oracle.row_size(t, 11008) % 16 == 0 else 14336        # rows must be 16-byte multiples (bulk copies)
    for (M, K) in [(1536, 4096), (1000, 2048), (264, k_sliced), (4096 + 24, 4096)]:
        W = weights(oracle, t, M, K, seed=M + K)
        Wd = dev(W)
        for n in ((1, 2, 3, 4, 5, 6, 7, 8) if M == 1536 else (2, 8, 5)):
            F = g.MM_GEMV | g.MM_GEMV_MMA
            assert g.mul_mat_plan(t, M, n, K, F) == g.MM_GEMV
            X = rng.uniform(-1, 1, (n, K)).astype(np.float32)
            Y = g.mul_mat(t, Wd, dev(X), M, n, K, flags=F).cpu().numpy()[0, 0]
            assert np.isfinite(Y).all()
            assert O.nmse(Y, oracle.mul_mat(t, W, X.reshape(-1), M, n, K)) < TOL, (M, K, n)
            Y2 = g.mul_mat(t, Wd, dev(X), M, n, K, flags=F | g.MM_SRC0_STATIC).cpu().numpy()[0, 0]
            assert np.array_equal(Y, Y2), (M, K, n, "not repeatable")
            if M == 1536 and n in (3, 8):
                for c in range(n):
                    y1 = g.mul_mat(t, Wd, dev(X[c]), M, 1, K, flags=F).cpu().numpy()[0, 0, 0]
                    assert np.array_equal(Y[c], y1), (n, c)
    # AUTO picks the mma kernel for 2 <= n <= 8 and leaves n = 1 on the dp4a kernel (same tolerance either way)
    M, K = 512, 4096
    W = weights(oracle, t, M, K, seed=5)
    X = rng.uniform(-1, 1, (4, K)).astype(np.float32)
    Ya = g.mul_mat(t, dev(W), dev(X), M, 4, K).cpu().numpy()[0, 0]
    Ym = g.mul_mat(t, dev(W), dev(X), M, 4, K, flags=g.MM_GEMV | g.MM_GEMV_MMA).cpu().numpy()[0, 0]
    assert np.array_equal(Ya, Ym)


@pytest.mark.parametrize("t", TYPES, ids=IDS)
def test_generic_shapes_vs_oracle(t, g, oracle):
    # the reference's own sweep: m=16, k=256, n=1..9 (tests/test-backend-ops.cpp:4005-4009), + ragged sizes
    cases = [(16, n, 256) for n in range(1, 10)] + [(5, 3, 512), (33, 17, 1024), (1, 1, 256)]
    if t in (O.Q4_0, O.Q8_0):
        cases += [(16, 1, 32), (7, 2, 96), (3, 5, 160)]
    for (M, N, K) in cases:
        W = weights(oracle, t, M, K, seed=7 * M + N + K)
        X = np.random.default_rng(M * N).uniform(-1, 1, N * K).astype(np.float32)
        Y = g.mul_mat(t, dev(W), dev(X), M, N, K, flags=g.MM_GENERIC).cpu().numpy()[0, 0]
        assert O.nmse(Y, oracle.mul_mat(t, W, X, M, N, K)) < TOL, (M, N, K)


@pytest.mark.parametrize("t", [O.Q4_0, O.Q4_K, O.Q6_K], ids=["q4_0", "q4_K", "q6_K"])
def test_batched_broadcast_strided(t, g, oracle):
    # bs = [3, 2], nr = [2, 2] as in tests/test-backend-ops.cpp:4017-4036, plus a padded (non-contiguous) src1
    import torch
    M, N, K = 16, 4, 256
    ne02, ne03, r2, r3 = 3, 2, 2, 2
    ne12, ne13 = ne02 * r2, ne03 * r3
    rb = oracle.row_size(t, K)
    W = weights(oracle, t, M * ne02 * ne03, K, seed=11)
    rng = np.random.default_rng(12)
    Xpad = rng.uniform(-1, 1, (ne13, ne12, N, K + 32)).astype(np.float32)
    X = np.ascontiguousarray(Xpad[..., :K])
    Xd = dev(Xpad)
    nb = (rb, rb * M, rb * M * ne02, (K + 32) * 4, (K + 32) * 4 * N, (K + 32) * 4 * N * ne12)
    Y = g.mul_mat(t, dev(W), Xd, M, N, K, batch=(ne02, ne03, ne12, ne13), nb=nb).cpu().numpy()
    for i13 in range(ne13):
        for i12 in range(ne12):
            w = W.reshape(ne03, ne02, M * rb)[i13 // r3, i12 // r2]
            want = oracle.mul_mat(t, w, X[i13, i12], M, N, K)
            assert O.nmse(Y[i13, i12], want) < TOL


@pytest.mark.parametrize("t", TYPES, ids=IDS)
def test_mul_mat_id_golden_and_oracle(t, g, oracle):
    z = np.load(G / f"mulmatid_{O.TYPE_NAMES[t]}.npz")
    ne, nu, nb1, ntok, M, K = (int(v) for v in z["cfg"])
    Y = g.mul_mat_id(t, dev(z["W"]), dev(z["X"]), dev(z["ids"]), M, K, ne, nu, nb1, ntok).cpu().numpy()
    assert O.nmse(Y, z["Y"]) < TOL
    # the reference's test shapes: m=512, k=256, n_mats 4/8, n_used 1/2/4, b broadcast or not, n 1/32
    rng = np.random.default_rng(5)
    for (ne, nu, bc, ntok) in [(4, 1, 0, 1), (4, 2, 0, 32), (8, 4, 1, 32), (8, 2, 1, 1), (8, 4, 0, 32)]:
        M, K = 512, 256
        nb1 = 1 if bc else nu
        W = weights(oracle, t, ne * M, K, seed=ne * 10 + nu)
        X = rng.uniform(-1, 1, ntok * nb1 * K).astype(np.float32)
        ids = np.stack([rng.permutation(ne) for _ in range(ntok)]).astype(np.int32)      # [ntok, ne]; first nu used (a strided view)
        Y = g.mul_mat_id(t, dev(W), dev(X), dev(ids), M, K, ne, nu, nb1, ntok).cpu().numpy()
        want = oracle.mul_mat_id(t, W, X, ids, M, K, ne, nu, nb1, ntok)
        assert O.nmse(Y, want) < TOL, (ne, nu, bc, ntok)


@pytest.mark.parametrize("t,M,K", [(O.Q4_K, 11008, 4096), (O.Q4_0, 4096, 4096), (O.Q8_0, 4096, 4096), (O.Q6_K, 4096, 4096), (O.Q5_K, 4096, 11008 // 256 * 256)],
                         ids=["q4_K-ffn", "q4_0-4096", "q8_0-4096", "q6_K-4096", "q5_K-11008"])
def test_full_size_properties(t, M, K, g, oracle):
    """BASELINE.json shapes: sampled rows against the oracle (rows are independent dot products), plus
    size-independent exact properties: power-of-two scaling of x scales y exactly; splitting M changes nothing."""
    import torch
    W = weights(oracle, t, M, K, seed=42, rng_blocks=True)
    X = np.random.default_rng(5678).uniform(-1, 1, K).astype(np.float32)
    Wd, Xd = dev(W), dev(X)
    assert g.mul_mat_plan(t, M, 1, K) == g.MM_GEMV
    Y = g.mul_mat(t, Wd, Xd, M, 1, K).cpu().numpy()[0, 0, 0]
    rows = np.random.default_rng(1).choice(M, 192, replace=False)
    rb = oracle.row_size(t, K)
    Wsub = np.concatenate([W[r * rb:(r + 1) * rb] for r in rows])
    want = oracle.mul_mat(t, Wsub, X, len(rows), 1, K)[0]
    assert O.nmse(Y[rows], want) < TOL
    Y4 = g.mul_mat(t, Wd, dev(X * 4.0), M, 1, K).cpu().numpy()[0, 0, 0]
    assert np.array_equal(Y4, Y * 4.0)
    half = (M // 2) // 16 * 16
    Ya = g.mul_mat(t, Wd[:half * rb], Xd, half, 1, K).cpu().numpy()[0, 0, 0]
    Yb = g.mul_mat(t, Wd[half * rb:], Xd, M - half, 1, K).cpu().numpy()[0, 0, 0]
    assert np.array_equal(np.concatenate([Ya, Yb]), Y)
    # generic kernel agrees bit-for-bit?  No (different summation order) -- but to round-off
    Yg = g.mul_mat(t, Wd, Xd, M, 1, K, flags=g.MM_GENERIC).cpu().numpy()[0, 0, 0]
    assert O.nmse(Yg, Y) < TOL


GEMM_TYPES = [O.Q4_0, O.Q8_0, O.Q4_K, O.Q5_K, O.Q6_K]


@pytest.mark.parametrize("t", GEMM_TYPES, ids=[O.TYPE_NAMES[t] for t in GEMM_TYPES])
def test_gemm_tcgen05_vs_oracle(t, g, oracle):
    """Tensor-core GEMM path (fp16 operands, f32 accumulation by wgmma).  Tolerances, stated: NMSE <= 1e-4 against the oracle (which
    itself carries the int8 activation-quantization noise), <= 2e-5 against the exact f64 product of the dequantized
    weights; the reference's own gate is 5e-4 (tests/test-backend-ops.cpp:1915-1917)."""
    # n = 9 .. 15 (the batches between the mat-vec kernels and a full 16-column tile) run on the tensor cores too
    for (M, N, K) in [(128, 16, 256), (256, 32, 512), (1000, 100, 1024), (384, 512, 2048), (130, 257, 768),
                      (64, 9, 512), (200, 13, 1024), (256, 15, 256), (300, 11, 2048), (128, 10, 4096), (520, 12, 2048), (96, 14, 2048)]:
        if g.mul_mat_plan(t, M, N, K, g.MM_GEMM) != g.MM_GEMM:
            assert t == O.Q6_K and K % 2048 != 0, (M, N, K)          # Q6_K rows are 16-byte multiples only when K % 2048 == 0 (TMA stride rule)
            continue
        assert g.mul_mat_plan(t, M, N, K) == g.MM_GEMM, (M, N, K)        # and AUTO picks it: no silent fall-back to the generic kernel
        W = weights(oracle, t, M, K, seed=3 * M + N + K)
        X = np.random.default_rng(N + K).uniform(-1, 1, N * K).astype(np.float32)
        Y = g.mul_mat(t, dev(W), dev(X), M, N, K, flags=g.MM_GEMM).cpu().numpy()[0, 0]
        assert np.isfinite(Y).all(), (M, N, K)
        assert O.nmse(Y, oracle.mul_mat(t, W, X, M, N, K)) < 1e-4, (M, N, K)
        assert O.nmse(Y, oracle.mul_mat(t, W, X, M, N, K, f64=True)) < 2e-5, (M, N, K)


@pytest.mark.parametrize("t", [O.Q8_0, O.Q4_K, O.Q6_K], ids=["q8_0", "q4_K", "q6_K"])
def test_gemm_full_size_properties(t, g, oracle):
    """BASELINE.json configs[2] (Q8_0 4096x4096, n_batch = 512) and its Q4_K twin: sampled rows against the oracle,
    and exact size-independent properties (column permutation equivariance, power-of-two scaling, repeatability)."""
    import torch
    M, N, K = 4096, 512, 4096
    W = weights(oracle, t, M, K, seed=77, rng_blocks=True)
    X = np.random.default_rng(5678).uniform(-1, 1, (N, K)).astype(np.float32)
    Wd, Xd = dev(W), dev(X)
    assert g.mul_mat_plan(t, M, N, K) == g.MM_GEMM
    Y = g.mul_mat(t, Wd, Xd, M, N, K).cpu().numpy()[0, 0]
    assert np.isfinite(Y).all()
    rows = np.random.default_rng(2).choice(M, 24, replace=False)
    rb = oracle.row_size(t, K)
    Wsub = np.concatenate([W[r * rb:(r + 1) * rb] for r in rows])
    want = oracle.mul_mat(t, Wsub, X.reshape(-1), len(rows), N, K, f64=True)
    assert O.nmse(Y[:, rows], want) < 2e-5
    Y2 = g.mul_mat(t, Wd, Xd, M, N, K).cpu().numpy()[0, 0]
    assert np.array_equal(Y, Y2)                                               # split-K hand-off is ordered: bitwise repeatable
    perm = np.random.default_rng(3).permutation(N)
    Yp = g.mul_mat(t, Wd, dev(X[perm]), M, N, K).cpu().numpy()[0, 0]
    assert np.array_equal(Yp, Y[perm])                                         # activation rows are independent
    # power-of-two scaling commutes with the fp16 rounding of the operands except for activations that become subnormal
    Y4 = g.mul_mat(t, Wd, dev(X * 0.25), M, N, K).cpu().numpy()[0, 0]
    assert O.nmse(Y4, Y * 0.25) < 1e-10
    # activations far outside the fp16 range: rows are pre-scaled by an exact power of two, the epilogue undoes it
    Xbig = X.copy(); Xbig[::2] *= 2.0 ** 20; Xbig[1::4] *= 2.0 ** -20
    Yb = g.mul_mat(t, Wd, dev(Xbig), M, N, K).cpu().numpy()[0, 0]
    assert np.isfinite(Yb).all()
    Yb[::2] *= 2.0 ** -20; Yb[1::4] *= 2.0 ** 20
    assert O.nmse(Yb, Y) < 1e-8


@pytest.mark.parametrize("t", [O.Q4_0, O.Q4_K, O.Q8_0], ids=["q4_0", "q4_K", "q8_0"])
def test_fused_epilogue_matches_separate_ops(t, g, oracle):
    """graph-level fusion used for the gpt-2 graph: MUL_MAT + ADD(bias) + GELU in one launch must write exactly what the
    three separate device ops write (which are themselves pinned by the reference's test-backend-ops)"""
    import torch
    M, K = 3072, 768 if t != O.Q4_K else 1024
    W = weights(oracle, t, M, K, seed=5)
    rng = np.random.default_rng(9)
    X = rng.uniform(-1, 1, K).astype(np.float32)
    bias = torch.from_numpy(rng.uniform(-0.5, 0.5, M).astype(np.float32)).cuda()
    Wd, Xd = dev(W), dev(X)
    y, y2, y3 = g.mul_mat_fused(t, Wd, Xd, M, K, bias, gelu=True)
    y_ref = g.mul_mat(t, Wd, Xd, M, 1, K).view(-1)
    assert torch.equal(y, y_ref)
    assert torch.equal(y2, y_ref + bias)
    assert torch.equal(y3, g.op_unary(0, y_ref + bias))
    assert O.nmse(y.cpu().numpy(), oracle.mul_mat(t, W, X, M, 1, K)[0]) < TOL


def test_fused_norm_affine_matches_separate_ops(g):
    import torch
    x = torch.randn(7, 768, device="cuda") * 3 + 0.5
    gain = torch.randn(768, device="cuda") * 0.02 + 1
    bias = torch.randn(768, device="cuda") * 0.02
    for rms in (False, True):
        y1, y2, y3 = g.op_norm_affine(x, gain, bias, 1e-5, rms=rms)
        n = g.op_norm(x, 1e-5, rms=rms)
        assert torch.equal(y1, n) and torch.equal(y2, n * gain) and torch.equal(y3, n * gain + bias)
        xd = x.double()
        ref = (xd / torch.sqrt((xd * xd).mean(-1, keepdim=True) + 1e-5)) if rms else ((xd - xd.mean(-1, keepdim=True)) / torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + 1e-5))
        assert O.nmse(y1.cpu().numpy(), ref.float().cpu().numpy()) < 1e-10


def test_fused_small_op_chains_match_separate_ops(g, oracle):
    """the token-graph fusions added for the gpt-2 decode path must write exactly what the separate ops write:
    SCALE -> DIAG_MASK_INF -> SOFT_MAX in one row pass; two float copies in one launch; MUL_MAT + bias + residual add in the epilogue"""
    import torch
    torch.manual_seed(3)
    for (heads, n1, n0, n_past) in [(12, 1, 37, 36), (12, 5, 9, 4), (3, 64, 200, 136), (1, 1, 1, 0), (12, 1, 1030, 1029)]:
        x = torch.randn(heads, n1, n0, device="cuda") * 4
        sep = g.op_soft_max(g.op_diag_mask_inf(g.op_scale(x, 0.125), n_past))
        fus = g.op_soft_max(x, scale=0.125, diag_n_past=n_past)
        assert torch.equal(sep, fus), (heads, n1, n0, n_past)
        ref = torch.softmax((x.double() * 0.125).masked_fill(torch.arange(n0, device="cuda")[None, None, :] > n_past + torch.arange(n1, device="cuda")[None, :, None], float("-inf")), -1)
        assert O.nmse(fus.cpu().numpy(), ref.float().cpu().numpy()) < 1e-10
    a, b = torch.randn(3, 768, device="cuda"), torch.randn(3, 768, device="cuda")
    da, db = torch.zeros(3, 768, device="cuda"), torch.zeros(3, 768, device="cuda", dtype=torch.float16)
    ea, eb = torch.zeros_like(da), torch.zeros_like(db)
    g.op_cpy2(a, da, b, db)
    g.op_cpy(a, ea); g.op_cpy(b, eb)
    assert torch.equal(da, ea) and torch.equal(db, eb) and torch.equal(da, a)
    M, K, t = 768, 3072, O.Q4_0
    W = weights(oracle, t, M, K, seed=15)
    rng = np.random.default_rng(16)
    X = rng.uniform(-1, 1, K).astype(np.float32)
    bias = torch.from_numpy(rng.uniform(-0.5, 0.5, M).astype(np.float32)).cuda()
    res = torch.from_numpy(rng.uniform(-2, 2, M).astype(np.float32)).cuda()
    y, y2, y3 = g.mul_mat_fused(t, dev(W), dev(X), M, K, bias, gelu=False, residual=res)
    y_ref = g.mul_mat(t, dev(W), dev(X), M, 1, K).view(-1)
    assert torch.equal(y, y_ref) and torch.equal(y2, y_ref + bias) and torch.equal(y3, (y_ref + bias) + res)
