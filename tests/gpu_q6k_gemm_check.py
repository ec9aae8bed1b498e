"""Run by tests/test_gpu_next_formats.py in a SUBPROCESS: the tensor-core GEMM path for Q6_K (variable-lead TMA boxes for the 2-byte-aligned
210-byte superblocks) against the oracle, incl. batches of 9..15 columns.  Exit code 0 = all checks passed."""
import os
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
    t = O.Q6_K
    rng = np.random.default_rng(61)
    for (M, N, K) in [(128, 16, 2048), (384, 100, 2048), (1000, 512, 4096), (4096, 512, 4096), (256, 9, 2048), (100, 15, 4096)]:
        assert g.mul_mat_plan(t, M, N, K) == g.MM_GEMM, (M, N, K)
        W = O.random_blocks(t, M * K // 256, rng)
        X = rng.uniform(-1, 1, N * K).astype(np.float32)
        Y = g.mul_mat(t, dev(W), dev(X), M, N, K).cpu().numpy()[0, 0]
        assert np.isfinite(Y).all()
        rows = rng.choice(M, min(M, 32), replace=False)
        rb = orc.row_size(t, K)
        Wsub = np.concatenate([W[r * rb:(r + 1) * rb] for r in rows])
        want = orc.mul_mat(t, Wsub, X, len(rows), N, K, f64=True)
        err = O.nmse(Y[:, rows], want)
        assert err < 2e-5, (M, N, K, err)
    torch.cuda.synchronize()
    print("q6_K tensor-core GEMM OK")


if __name__ == "__main__":
    main()
