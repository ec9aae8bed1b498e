"""Developer sweep: device time of the tensor-core (wgmma) GEMM (n = 512 etc.)"""
import json, sys
from pathlib import Path
import numpy as np, torch
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import ggml_b200 as g
NAMES = {v: k for k, v in g.TYPE_NAMES.items()}
for tn in ("q8_0", "q4_K", "q4_0", "q5_K"):
    t = NAMES[tn]
    for (M, N, K) in [(4096, 512, 4096), (11008, 512, 4096), (4096, 128, 4096), (4096, 32, 4096), (32000, 512, 4096)]:
        if g.mul_mat_plan(t, M, N, K, g.MM_GEMM) != g.MM_GEMM:
            print(json.dumps({"type": tn, "M": M, "N": N, "K": K, "skip": "not eligible"})); continue
        rb = g.row_size(t, K)
        W = torch.randint(0, 256, (M * rb,), dtype=torch.uint8, device="cuda")
        X = torch.rand(N * K, device="cuda") * 2 - 1
        Y = torch.empty((1, 1, N, M), device="cuda")
        for _ in range(3):
            g.mul_mat(t, W, X, M, N, K, flags=g.MM_GEMM, out=Y)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 30
        e0.record()
        for _ in range(reps):
            g.mul_mat(t, W, X, M, N, K, flags=g.MM_GEMM, out=Y)
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1000 / reps
        print(json.dumps({"type": tn, "M": M, "N": N, "K": K, "us": round(us, 1), "TFLOPs": round(2.0 * M * N * K / us / 1e6, 1)}), flush=True)
