"""GPU: the SURVEY §8f-2 formats (Q4_1, Q5_0, Q5_1, Q2_K, Q3_K, IQ4_NL, IQ4_XS) on the superblock and generic mat-vec / tensor-core GEMM /
MUL_MAT_ID / dequantize kernels, Q6_K and the edge shapes of the tensor-core GEMM (mmq_tc2.cu).

Each check runs in a subprocess (own CUDA context), which keeps a device fault in one of them from taking the rest of the suite down with it."""
import subprocess
import sys
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def test_next_formats_parity_subprocess():
    p = subprocess.run([sys.executable, str(ROOT / "tests" / "gpu_next_formats_check.py")], capture_output=True, text=True, timeout=300)
    print(p.stdout[-2000:])
    assert p.returncode == 0, (p.stdout + p.stderr)[-3000:]


def test_q6k_gemm_subprocess():
    p = subprocess.run([sys.executable, str(ROOT / "tests" / "gpu_q6k_gemm_check.py")], capture_output=True, text=True, timeout=200)
    print(p.stdout[-2000:])
    assert p.returncode == 0, (p.stdout + p.stderr)[-3000:]


def test_gemm_edge_shapes_subprocess():
    p = subprocess.run([sys.executable, str(ROOT / "tests" / "gpu_tc2_check.py")], capture_output=True, text=True, timeout=300)
    print(p.stdout[-2000:])
    assert p.returncode == 0, (p.stdout + p.stderr)[-3000:]


def test_mul_mat_id_expert_grouped_subprocess():
    """MUL_MAT_ID with the rows grouped per expert on the device and multiplied on the tensor-core GEMM kernel (opt-in GGML_B200_MMID_GROUPED=1),
    in its own process"""
    import os
    env = dict(os.environ, GGML_B200_MMID_GROUPED="1")
    p = subprocess.run([sys.executable, str(ROOT / "tests" / "gpu_mmid_grouped_check.py"), "--time"], capture_output=True, text=True, timeout=300, env=env)
    print(p.stdout[-2000:])
    assert p.returncode == 0, (p.stdout + p.stderr)[-3000:]
