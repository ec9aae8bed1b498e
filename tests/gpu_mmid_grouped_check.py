"""Run in a SUBPROCESS with GGML_B200_MMID_GROUPED=1: MUL_MAT_ID with the rows grouped per expert on the device and multiplied on the
tensor-core GEMM kernel (mmq_tc2.cu, GROUPED mode) against the CPU oracle; --time prints the device time of the Mixtral-like case (8 experts, 2 used,
512 tokens, 4096 x 4096 Q4_K) for the grouped path and for the per-pair mat-vec path.  Exit code 0 = all checks passed."""
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
    assert os.environ.get("GGML_B200_MMID_GROUPED") == "1"
    g.lib()
    orc = O.Oracle()
    rng = np.random.default_rng(31)
    for (t, ne, nu, bc, ntok, M, K) in [(O.Q4_K, 8, 2, 0, 512, 1024, 1024), (O.Q8_0, 4, 1, 0, 100, 512, 512), (O.Q4_0, 8, 4, 1, 64, 300, 768), (O.Q6_K, 8, 2, 0, 129, 256, 2048),
                                        (O.Q4_K, 16, 4, 0, 37, 640, 256)]:
        nb1 = 1 if bc else nu
        W = O.random_blocks(t, ne * M * K // orc.blck_size(t), rng)
        X = rng.uniform(-1, 1, ntok * nb1 * K).astype(np.float32)
        # skewed routing: some experts get many tokens, some none
        p = rng.dirichlet(np.ones(ne) * 0.5)
        ids = np.stack([rng.choice(ne, size=nu, replace=False, p=p) for _ in range(ntok)]).astype(np.int32)
        Y = g.mul_mat_id(t, dev(W), dev(X), dev(ids), M, K, ne, nu, nb1, ntok).cpu().numpy()
        assert np.isfinite(Y).all()
        want = orc.mul_mat_id(t, W, X, ids, M, K, ne, nu, nb1, ntok)
        err = O.nmse(Y, want)
        assert err < 1e-4, (O.TYPE_NAMES[t], ne, nu, ntok, M, K, err)          # fp16 operands on the tensor-core path (reference gate 5e-4)
        print(f"ok grouped mul_mat_id {O.TYPE_NAMES[t]} experts={ne} used={nu} tokens={ntok} {M}x{K} nmse {err:.2e}", flush=True)
    if "--time" in sys.argv:
        t, ne, nu, ntok, M, K = O.Q4_K, 8, 2, 512, 4096, 4096
        W = dev(O.random_blocks(t, ne * M * K // 256, rng))
        X = dev(rng.uniform(-1, 1, ntok * nu * K).astype(np.float32))
        ids = dev(np.stack([rng.permutation(ne)[:nu] for _ in range(ntok)]).astype(np.int32))
        for _ in range(3):
            g.mul_mat_id(t, W, X, ids, M, K, ne, nu, nu, ntok)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            g.mul_mat_id(t, W, X, ids, M, K, ne, nu, nu, ntok)
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 100
        print(f"time grouped mul_mat_id q4_K 8x2 experts, 512 tokens, 4096x4096: {us:.1f} us = {2.0 * ntok * nu * M * K / us / 1e6:.0f} TFLOP/s", flush=True)
    print("grouped mul_mat_id OK")


if __name__ == "__main__":
    main()
