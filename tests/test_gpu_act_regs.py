"""GPU: the superblock mat-vec's activation-stationary consume path (Q4_K / Q5_K, n = 1, K <= 4096, independent launches on 4-warp CTAs;
GGML_B200_SB_ACT_REGS=1, the default) against the shared-memory consume path it replaces (GGML_B200_SB_ACT_REGS=0): bit-identical outputs
for ragged row counts, K = 256 .. 4096 and the fused bias / GELU / residual epilogue, dependent launches (8-warp CTAs, which keep the
shared-memory paths) unchanged by the switch, all within the usual tolerance of the CPU oracle.  Each arm runs in its own process (the
switch is read once)."""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import oracle as O  # noqa: E402

# (name, type, M, K, mode): mode "ind" = SRC0|SRC1_STATIC (4-warp CTAs), "dep" = SRC0_STATIC (8-warp CTAs; with M, K >= 2048 the
# two-row form), "gelu" / "res" = the fused epilogue entry point with SRC0|SRC1_STATIC
CASES = [
    ("q4k_headline_ind", O.Q4_K, 11008, 4096, "ind"),
    ("q4k_headline_dep", O.Q4_K, 11008, 4096, "dep"),
    ("q5k_ragged_ind", O.Q5_K, 4099, 4096, "ind"),
    ("q5k_ragged_dep", O.Q5_K, 4099, 4096, "dep"),
    ("q4k_k256_ind", O.Q4_K, 1003, 256, "ind"),
    ("q4k_k256_dep", O.Q4_K, 1003, 256, "dep"),
    ("q5k_k1024_dep", O.Q5_K, 777, 1024, "dep"),
    ("q4k_k3072_ind", O.Q4_K, 2050, 3072, "ind"),
    ("q4k_fused_gelu", O.Q4_K, 2051, 4096, "gelu"),
    ("q5k_fused_res", O.Q5_K, 1001, 4096, "res"),
]


def _inputs(i, t, M, K):
    rng = np.random.default_rng(4200 + i)
    W = O.random_blocks(t, M * K // 256, rng)
    X = rng.uniform(-1, 1, K).astype(np.float32)
    bias = rng.uniform(-1, 1, M).astype(np.float32)
    res = rng.uniform(-1, 1, M).astype(np.float32)
    return W, X, bias, res


def _child(out_path):
    import torch
    import ggml_b200 as g
    torch.cuda.set_device(0)
    out = {}
    for i, (name, t, M, K, mode) in enumerate(CASES):
        W, X, bias, res = (torch.from_numpy(a).cuda() for a in _inputs(i, t, M, K))
        if mode in ("ind", "dep"):
            flags = g.MM_SRC0_STATIC | (g.MM_SRC1_STATIC if mode == "ind" else 0)
            assert g.mul_mat_plan(t, M, 1, K, flags) == g.MM_GEMV
            y = g.mul_mat(t, W, X, M, 1, K, flags=flags)
            out[name] = y.view(-1).cpu().numpy()
        else:
            # ggml_b200.mul_mat_fused with the independent-launch flags
            L = g.lib()
            Y, Y2, Y3 = (torch.empty(M, dtype=torch.float32, device="cuda") for _ in range(3))
            a = g.mul_mat_args(t, W, X, Y, M, 1, K, flags=g.MM_SRC0_STATIC | g.MM_SRC1_STATIC)
            ep = g.Epilogue()
            ep.bias, ep.dst_bias, ep.unary, ep.dst_unary = bias.data_ptr(), Y2.data_ptr(), (2 if mode == "res" else 1), Y3.data_ptr()
            ep.residual = res.data_ptr() if mode == "res" else None
            g.check(L.ggml_b200_mul_mat_fused(C.byref(a), C.byref(ep), torch.cuda.current_stream().cuda_stream), "ggml_b200_mul_mat_fused")
            out[name], out[name + "_y2"], out[name + "_y3"] = Y.cpu().numpy(), Y2.cpu().numpy(), Y3.cpu().numpy()
    torch.cuda.synchronize()
    np.savez(out_path, **out)


def _run_arm(tmp_path, areg):
    out = tmp_path / f"arm{areg}.npz"
    env = dict(os.environ, GGML_B200_SB_ACT_REGS=str(areg))
    p = subprocess.run([sys.executable, __file__, "--child", str(out)], env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, (p.stdout + p.stderr)[-3000:]
    return dict(np.load(out))


@pytest.mark.gpu
def test_act_regs_bit_identical_to_shared_memory_consume(tmp_path, oracle):
    old, new = _run_arm(tmp_path, 0), _run_arm(tmp_path, 1)
    assert sorted(old) == sorted(new)
    for k in old:
        assert np.array_equal(old[k].view(np.uint32), new[k].view(np.uint32)), k
    for i, (name, t, M, K, mode) in enumerate(CASES):
        W, X, bias, res = _inputs(i, t, M, K)
        want = oracle.mul_mat(t, W, X, M, 1, K).reshape(-1)
        err = O.nmse(new[name], want)
        assert err < 1e-10, (name, err)
        if mode == "res":
            assert np.array_equal(new[name + "_y3"], (new[name] + bias) + res), name
        if mode in ("gelu", "res"):
            assert np.array_equal(new[name + "_y2"], new[name] + bias), name


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--child":
        _child(sys.argv[2])
