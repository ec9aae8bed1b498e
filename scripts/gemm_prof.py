"""Developer aid: one batched mul_mat shape on the tensor-core path, timed with CUDA events over CUDA-graph replays (and a plain warm loop for ncu).
usage: python scripts/gemm_prof.py TYPE M N K [--ncu]"""
import os
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import ggml_b200 as g  # noqa: E402
from oracle import oracle as O  # noqa: E402

t = {v: k for k, v in g.TYPE_NAMES.items()}[sys.argv[1]]
M, N, K = (int(v) for v in sys.argv[2:5])
rng = np.random.default_rng(1)
nbuf = int(os.environ.get("GEMM_PROF_NBUF", "4"))      # 4 matrices stay L2-resident at 4096^2; bench.py rotates enough of them to stream from HBM
Ws = [torch.from_numpy(O.random_blocks(t, M * K // O.Oracle().blck_size(t), rng)).cuda() for _ in range(nbuf)]
X = torch.from_numpy(rng.uniform(-1, 1, N * K).astype(np.float32)).cuda()
Ys = [torch.empty((1, 1, N, M), device="cuda") for _ in range(nbuf)]
F = g.MM_SRC0_STATIC | g.MM_SRC1_STATIC
assert g.mul_mat_plan(t, M, N, K) == g.MM_GEMM


def sweep():
    for i in range(nbuf):
        g.mul_mat(t, Ws[i], X, M, N, K, out=Ys[i], flags=F)


for _ in range(3):
    sweep()
torch.cuda.synchronize()
if "--ncu" in sys.argv:
    sweep()
    torch.cuda.synchronize()
    sys.exit(0)
graph = torch.cuda.CUDAGraph()
with torch.cuda.graph(graph):
    sweep()
for _ in range(3):
    graph.replay()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(50):
    graph.replay()
e1.record()
torch.cuda.synchronize()
us = e0.elapsed_time(e1) * 1e3 / (50 * nbuf)
tun = {k: v for k, v in os.environ.items() if k.startswith("GGML_B200_")}
print(f"{g.TYPE_NAMES[t]} {M}x{N}x{K}: {us:.2f} us per mul_mat = {2.0 * M * N * K / us / 1e6:.0f} TFLOP/s  {tun}", flush=True)
