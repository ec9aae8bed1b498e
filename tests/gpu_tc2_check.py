"""Run in a SUBPROCESS (own CUDA context, short timeout): the tensor-core GEMM (mmq_tc2.cu, wgmma) against the f64 product of the oracle's
dequantized weights on shapes that exercise: tiles whose second warpgroup has no valid rows (M <= 128, including the Q8_0 shapes that turn the
raw-weight ring over fastest), split-K, both tile widths (BN = 64 / 128), ragged N / M tails, K-quant and 2-byte-aligned formats; and that a
repeated launch is bitwise identical.  Exit code 0 = all checks passed."""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import ggml_b200 as g  # noqa: E402
from oracle import oracle as O  # noqa: E402


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def main():
    g.lib()
    orc = O.Oracle()
    rng = np.random.default_rng(22)
    cases = [(O.Q8_0, 256, 64, 256), (O.Q8_0, 512, 512, 1024), (O.Q4_K, 4096, 512, 4096), (O.Q4_0, 300, 100, 512), (O.Q5_K, 1000, 257, 2048),
             (O.Q6_K, 640, 130, 2048), (O.Q8_0, 200, 40, 768), (O.Q4_K, 11008, 96, 1024), (O.Q3_K, 520, 70, 2048), (O.Q5_0, 260, 33, 512),
             (O.Q8_0, 128, 10, 4096), (O.Q8_0, 128, 64, 4096), (O.Q8_0, 100, 300, 8192), (O.Q8_0, 4096, 512, 4096)]
    for (t, M, N, K) in cases:
        assert g.mul_mat_plan(t, M, N, K) == g.MM_GEMM, (O.TYPE_NAMES[t], M, N, K)     # (rows must be 16-byte multiples: Q3_K / Q6_K need K % 2048 == 0)
        W = O.random_blocks(t, M * K // orc.blck_size(t), rng)
        X = rng.uniform(-1, 1, N * K).astype(np.float32)
        Wd, Xd = dev(W), dev(X)
        Y = g.mul_mat(t, Wd, Xd, M, N, K).cpu().numpy()[0, 0]
        assert np.isfinite(Y).all(), (O.TYPE_NAMES[t], M, N, K)
        rows = np.sort(rng.choice(M, min(M, 40), replace=False))
        rows[0], rows[-1] = 0, M - 1
        rb = orc.row_size(t, K)
        Wsub = np.concatenate([W[r * rb:(r + 1) * rb] for r in rows])
        want = orc.mul_mat(t, Wsub, X, len(rows), N, K, f64=True)
        err = O.nmse(Y[:, rows], want)
        assert err < 2e-5, (O.TYPE_NAMES[t], M, N, K, err)
        Y2 = g.mul_mat(t, Wd, Xd, M, N, K).cpu().numpy()[0, 0]
        assert np.array_equal(Y, Y2), ("not repeatable", O.TYPE_NAMES[t], M, N, K)
        print(f"ok {O.TYPE_NAMES[t]} {M}x{N}x{K} nmse {err:.2e}", flush=True)
    print("tensor-core GEMM edge shapes OK")


if __name__ == "__main__":
    main()
