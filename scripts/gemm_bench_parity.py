"""Developer aid: the bench's batched-GEMM leg (NBUF distinct matrices, CUDA-graph replays of PDL-overlapped launches flagged
SRC0|SRC1_STATIC, weights streaming from HBM) with EVERY element of every output checked against the exact f64 product.
usage: python scripts/gemm_bench_parity.py TYPE M N K [--plain] [--noflags]
  --plain    plain stream launches instead of a CUDA graph        --noflags  MM_AUTO instead of the static flags"""
import os
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
import ggml_b200 as g  # noqa: E402

t = {v: k for k, v in g.TYPE_NAMES.items()}[sys.argv[1]]
M, N, K = (int(v) for v in sys.argv[2:5])
wb = bench.weight_bytes(K, M, t)
nbuf = max(2, int(np.ceil(260e6 / wb)))
Ws = bench.make_weights(torch, t, nbuf, K, M, 11)
X = torch.rand(N * K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5678)) * 2 - 1
Ys = [torch.empty((1, 1, N, M), dtype=torch.float32, device="cuda") for _ in range(nbuf)]
F = g.MM_AUTO if "--noflags" in sys.argv else (g.MM_SRC0_STATIC | g.MM_SRC1_STATIC)


def sweep():
    for i in range(nbuf):
        g.mul_mat(t, Ws[i], X, M, N, K, out=Ys[i], flags=F)


sweep()
torch.cuda.synchronize()
if "--plain" in sys.argv:
    for _ in range(20):
        sweep()
    torch.cuda.synchronize()
else:
    timer = bench.Timer(torch)
    s, reps = timer.time_graph(sweep, min_seconds=0.05)
    print(f"{s / nbuf * 1e6:.2f} us per mul_mat over {reps} replays of {nbuf} matrices", flush=True)
Xd = X.view(N, K).double()


def check(label, verbose=True):
    bad, wrong_rows = 0, {}
    for i in range(nbuf):
        Wf = g.dequantize(t, Ws[i], M * K).view(M, K).double()
        exact = Xd @ Wf.T
        scale = exact.abs().mean().item()
        err = (Ys[i][0, 0].double() - exact).abs()
        wrong = err > 6e-3 * scale
        if wrong.any():
            bad += 1
            idx = wrong.nonzero()
            cols, rows = idx[:, 0].cpu().numpy(), idx[:, 1].cpu().numpy()
            wrong_rows[i] = sorted(set(rows.tolist()))
            if verbose and bad <= 3:
                print(f"  [{label}] matrix {i}: {len(rows)} elements off by up to {err.max().item() / scale:.3f} x typical; distinct rows {len(wrong_rows[i])}: {wrong_rows[i][:10]}, "
                      f"cols {cols.min()}..{cols.max()} ({len(set(cols.tolist()))} distinct)", flush=True)
    return bad, wrong_rows


bad, rows_a = check("overlapped")
if "--serial" in sys.argv:
    # the same launches again, one at a time with a device synchronisation after each: a race between overlapping launches disappears,
    # a data-dependent decode error stays on the same rows
    for Y in Ys:
        Y.zero_()
    for i in range(nbuf):
        g.mul_mat(t, Ws[i], X, M, N, K, out=Ys[i], flags=F)
        torch.cuda.synchronize()
    bad_s, rows_s = check("serial")
    same = sum(1 for i in rows_s if rows_a.get(i) == rows_s[i])
    print(f"serial re-run: {bad_s} of {nbuf} matrices wrong ({same} with exactly the rows of the overlapped run)", flush=True)
tun = {k: v for k, v in os.environ.items() if k.startswith("GGML_B200_")}
print(("CLEAN" if bad == 0 else f"BAD ({bad} of {nbuf} matrices)"), g.TYPE_NAMES[t], M, N, K, sys.argv[5:], tun, flush=True)
