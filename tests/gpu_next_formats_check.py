"""Run by tests/test_gpu_next_formats.py in a SUBPROCESS (its own CUDA context): parity of the SURVEY §8f-2 formats
(Q4_1, Q5_0, Q5_1, Q2_K, Q3_K, IQ4_NL, IQ4_XS) through the C ABI — dequantize bit-exact, generic MUL_MAT and MUL_MAT_ID within NMSE 1e-10 of the
oracle and of the reference's golden vectors.  Exit code 0 = all checks passed."""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import ggml_b200 as g  # noqa: E402
from oracle import oracle as O  # noqa: E402

G = ROOT / "tests" / "golden"
TOL = 1e-10


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def main():
    g.lib()
    orc = O.Oracle()
    done = []
    for t in tuple(O.NEXT_TYPES) + tuple(O.IQ_TYPES):          # + the grid i-quants (generic kernels)
        name = O.TYPE_NAMES[t]
        z = np.load(G / f"quant_{name}.npz")
        for blocks, want in ((z["blocks"], z["deq"]), (z["rnd_blocks"], z["rnd_deq"])):
            got = g.dequantize(t, dev(blocks), want.size).cpu().numpy()
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), ("dequantize f32", name)
            got16 = g.dequantize(t, dev(blocks), want.size, dtype=torch.float16).cpu().numpy()
            assert np.array_equal(got16.view(np.uint16), want.astype(np.float16).view(np.uint16)), ("dequantize f16", name)
        z = np.load(G / f"mulmat_{name}.npz")
        for ci in range(int(z["ncases"])):
            M, N, K = (int(v) for v in z[f"shape{ci}"])
            for flags in (g.MM_AUTO, g.MM_GENERIC):           # AUTO = superblock kernel (n <= 8) / tensor-core GEMM (n >= 9) where eligible
                Y = g.mul_mat(t, dev(z[f"W{ci}"]), dev(z[f"X{ci}"]), M, N, K, flags=flags).cpu().numpy()[0, 0]
                tol = 1e-4 if g.mul_mat_plan(t, M, N, K, flags) == g.MM_GEMM else TOL     # fp16 operands on the tensor-core path
                assert O.nmse(Y, z[f"Y{ci}"]) < tol, ("golden mul_mat", name, ci, flags)
        rng = np.random.default_rng(900 + t)
        for (M, N, K) in [(16, 1, 256), (33, 5, 1024), (1000, 2, 4096), (257, 17, 512), (4096, 1, 4096), (1536, 8, 2048)] + ([(7, 2, 96), (16, 3, 160)] if orc.blck_size(t) == 32 else []):
            W = O.random_blocks(t, M * K // orc.blck_size(t), rng)
            X = rng.uniform(-1, 1, N * K).astype(np.float32)
            want = orc.mul_mat(t, W, X, M, N, K)
            for flags in (g.MM_AUTO, g.MM_GENERIC):
                Y = g.mul_mat(t, dev(W), dev(X), M, N, K, flags=flags).cpu().numpy()[0, 0]
                tol = 1e-4 if g.mul_mat_plan(t, M, N, K, flags) == g.MM_GEMM else TOL
                assert O.nmse(Y, want) < tol, ("oracle mul_mat", name, M, N, K, flags)
        # tensor-core path (fp16 operands): against the exact product of the dequantized weights, sampled rows
        for (M, N, K) in [(512, 64, 2048), (1000, 512, 4096)]:
            if g.mul_mat_plan(t, M, N, K) != g.MM_GEMM:
                continue
            W = O.random_blocks(t, M * K // orc.blck_size(t), rng)
            X = rng.uniform(-1, 1, N * K).astype(np.float32)
            Y = g.mul_mat(t, dev(W), dev(X), M, N, K).cpu().numpy()[0, 0]
            assert np.isfinite(Y).all(), ("gemm finite", name, M, N, K)
            rows = rng.choice(M, 24, replace=False)
            rb = orc.row_size(t, K)
            Wsub = np.concatenate([W[r * rb:(r + 1) * rb] for r in rows])
            want = orc.mul_mat(t, Wsub, X, len(rows), N, K, f64=True)
            assert O.nmse(Y[:, rows], want) < 2e-5, ("gemm", name, M, N, K)
        z = np.load(G / f"mulmatid_{name}.npz")
        ne, nu, nb1, ntok, M, K = (int(v) for v in z["cfg"])
        Y = g.mul_mat_id(t, dev(z["W"]), dev(z["X"]), dev(z["ids"]), M, K, ne, nu, nb1, ntok).cpu().numpy()
        assert O.nmse(Y, z["Y"]) < TOL, ("golden mul_mat_id", name)
        done.append(name)
    # the Q8_1 "s" section of the activation record (block_q8_1.s = fp16(d_unrounded * sum of codes)), used by Q4_1 / Q5_1
    K = 3072
    rng = np.random.default_rng(8)
    X = np.stack([rng.uniform(-1, 1, K), rng.standard_normal(K) * 7, np.zeros(K), np.round(rng.uniform(-127, 127, K)) / 2]).astype(np.float32)
    rec = g.quantize_activations(O.Q4_1, dev(X)).cpu().numpy()
    bs_off = (K + 15) & ~15
    d_off = bs_off + ((K // 16 * 2 + 15) & ~15)
    s_off = d_off + ((K // 32 * 4 + 15) & ~15)
    for r in range(X.shape[0]):
        want = orc.quantize(O.Q8_1, X[r]).reshape(-1, 36)
        assert np.array_equal(rec[r, :K].view(np.int8), want[:, 4:].reshape(-1).view(np.int8)), ("q8_1 codes", r)
        assert np.array_equal(rec[r, d_off:d_off + K // 32 * 4].copy().view(np.float32), want[:, :2].copy().view(np.float16).astype(np.float32).reshape(-1)), ("q8_1 d", r)
        assert np.array_equal(rec[r, s_off:s_off + K // 32 * 4].copy().view(np.float32), want[:, 2:4].copy().view(np.float16).astype(np.float32).reshape(-1)), ("q8_1 s", r)
    torch.cuda.synchronize()
    print("next formats OK:", " ".join(done), "+ q8_1 activation record")


if __name__ == "__main__":
    main()
