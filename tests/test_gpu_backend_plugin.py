"""GPU: the ggml backend plug-in (libggml-b200.so) driven by the UNMODIFIED reference harness.

oracle/_ref holds the reference compiled from /root/reference (libggml-base/-cpu, tests/test-backend-ops.cpp,
examples/gpt-2); the plug-in is discovered through the reference's own dynamic loader ($GGML_BACKEND_PATH,
src/ggml-backend-reg.cpp:578-581).  test-backend-ops compares every MUL_MAT / MUL_MAT_ID case against ggml-cpu
with its NMSE <= 5e-4 gate (tests/test-backend-ops.cpp:1915-1917) — the reference's own parity contract."""
import re
import subprocess

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def plugin():
    import ggml_b200
    if not ggml_b200.BACKEND_SO.exists():
        pytest.fail(f"{ggml_b200.BACKEND_SO} missing: run __graft_entry__.build() where the ggml headers are available")
    if not (O.REF_DIR / "test-backend-ops").exists():
        pytest.fail("oracle/_ref/test-backend-ops missing (built by oracle/Makefile in the build container)")
    return ggml_b200.BACKEND_SO


def run_tbo(plugin, *args, timeout=900):
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(plugin)
    p = subprocess.run([str(O.REF_DIR / "test-backend-ops"), *args], env=env, capture_output=True, text=True, timeout=timeout)
    return p.returncode, p.stdout + p.stderr


@pytest.mark.parametrize("op", ["MUL_MAT", "MUL_MAT_ID"])
def test_reference_test_backend_ops(plugin, op):
    rc, out = run_tbo(plugin, "test", "-o", op, "-b", "B2000")
    tail = "\n".join(out.splitlines()[-15:])
    assert rc == 0, tail
    m = re.search(r"(\d+)/(\d+) tests passed", out)
    assert m and m.group(1) == m.group(2) and int(m.group(2)) > 0, tail
    assert "Backend B2000" in out and "FAIL" not in out, tail
    # the cases this backend claims (not "not supported") must include every hot-path type
    for tname in ("q4_0", "q8_0", "q4_K", "q5_K", "q6_K"):
        ok_lines = [l for l in out.splitlines() if f"type_a={tname}," in l and "type_b=f32" in l and "OK" in l]
        assert ok_lines, f"no executed {op} case for {tname}"


def test_plugin_vs_cpu_backend_large(plugin):
    """Through the reference's graph + backend API (tensor_set -> graph_compute -> tensor_get) at BASELINE sizes."""
    ref = O.Ref()
    assert ref.load_backend(plugin)
    assert "B2000" in ref.devices()
    rng = np.random.default_rng(1234)
    for t, M, N, K in [(O.Q4_K, 11008, 1, 4096), (O.Q4_0, 4096, 1, 4096), (O.Q8_0, 4096, 4, 4096), (O.Q6_K, 1024, 2, 4096), (O.Q5_K, 512, 1, 2048)]:
        W = ref.quantize(t, rng.uniform(-1, 1, M * K).astype(np.float32), M, K)       # the reference's own quantizer
        X = np.random.default_rng(5678).uniform(-1, 1, N * K).astype(np.float32)
        Yg, _ = ref.mul_mat(t, W, X, M, N, K, dev="B2000")
        Yc, _ = ref.mul_mat(t, W, X, M, N, K, dev="CPU", threads=16)
        assert O.nmse(Yg, Yc) < 1e-10, (O.TYPE_NAMES[t], M, N, K)


@pytest.mark.parametrize("op", ["GET_ROWS", "ADD", "MUL", "NORM", "RMS_NORM", "SCALE", "DIAG_MASK_INF", "SOFT_MAX", "GELU", "SILU", "CPY", "CONT", "DUP",
                                "FLASH_ATTN_EXT", "DIV", "TANH", "NEG", "ABS", "GELU_QUICK", "SIGMOID", "EXP", "RELU", "STEP"])
def test_reference_test_backend_ops_small_ops(plugin, op):
    """the ops either side of the mat-mul in the gpt-2 graph (SURVEY.md §8f-1) and the other binary and unary ops the plug-in accepts
    (SQR, SQRT, SIN and COS run in tests/test_gpu_rwkv.py and tests/test_gpu_sam.py; the reference's sweep has no SUB case, which
    tests/test_gpu_core_ops.py covers), gated by the reference's own per-op tolerances (default NMSE 1e-7; CPY/SOFT_MAX 1e-6)"""
    rc, out = run_tbo(plugin, "test", "-o", op, "-b", "B2000")
    tail = "\n".join(out.splitlines()[-25:])
    assert rc == 0 and "FAIL" not in out, tail
    assert any("OK" in l and "not supported" not in l for l in out.splitlines() if l.strip().startswith(op + "(")), f"no executed {op} case\n{tail}"


def test_reference_test_mul_mat_route_b(plugin):
    """tests/test-mul-mat.cpp compiled UNMODIFIED with -DGGML_USE_CUDA binds ggml_backend_cuda_init, which this
    library exports (include/ggml-cuda.h ABI): exact F32 golden matrix through MUL_MAT + CONT + TRANSPOSE."""
    exe = O.REF_DIR / "test-mul-mat-b200"
    if not exe.exists():
        pytest.fail("oracle/_ref/test-mul-mat-b200 missing (make -C oracle b200bins)")
    p = subprocess.run([str(exe)], env=O.ref_env(), capture_output=True, text=True, timeout=120)
    out = p.stdout + p.stderr
    assert p.returncode == 0 and out.count("PASSED") >= 2 and "FAILED" not in out, out[-1500:]
    assert "using CUDA backend" in out, out[-1500:]


def test_split_buffer_mul_mat(plugin):
    """The reference's multi-GPU entry: weights in the buffer type returned by get_proc_address("ggml_backend_split_buffer_type")
    (src/ggml-cuda/ggml-cuda.cu:1000, 3374-3380), rows sharded over every visible device, MUL_MAT through the vtable.  With one GPU
    the split is trivial (plumbing check: init_tensor / scatter set_tensor / gather get_tensor / compute); with more it is the
    single-process multi-device path (peer stores into the main device's dst over NVLink for n = 1, staged peer copies for batches).
    The result must equal the 1-device result (bit-identical wherever both run the same kernel: rows are independent) and the oracle."""
    import torch
    ref = O.Ref()
    assert ref.load_backend(plugin)
    ndev = torch.cuda.device_count()
    orc = O.Oracle()
    rng = np.random.default_rng(77)
    cases = [(O.Q4_K, 11008, 1, 4096), (O.Q8_0, 4096, 1, 4096), (O.Q6_K, 1000, 1, 2048), (O.Q4_0, 4096, 4, 4096), (O.Q4_K, 2048, 64, 1024), (O.Q4_K, 28672, 1, 8192)]
    splits = [None] + ([[3.0, 1.0] + [0.0] * (ndev - 2)] if ndev >= 2 else [])
    for t, M, N, K in cases:
        W = O.random_blocks(t, M * K // orc.blck_size(t), rng)
        X = rng.uniform(-1, 1, N * K).astype(np.float32)
        Y1, _ = ref.mul_mat(t, W, X, M, N, K, dev="B2000")
        for ts in splits:
            Ys, _ = ref.mul_mat_split(t, W, X, M, N, K, dev="B2000", main_device=0, tensor_split=ts)
            if N <= 8 and not (N == 1 and K >= 12288):
                assert np.array_equal(Ys, Y1[0, 0]), (O.TYPE_NAMES[t], M, N, K, ts)
            elif N == 1:
                # long rows: one device runs the mma kernel (api.cu::mma_wanted), the split path the fused-gather dp4a kernel: same integer
                # dots, different f32 summation order
                assert O.nmse(Ys, Y1[0, 0]) < 1e-12, (O.TYPE_NAMES[t], M, N, K, ts)
            else:
                assert O.nmse(Ys, Y1[0, 0]) < 1e-6, (O.TYPE_NAMES[t], M, N, K, ts)       # tile / split-K grouping differs per shard
        rows = rng.choice(M, 64, replace=False)
        rb = orc.row_size(t, K)
        want = orc.mul_mat(t, np.concatenate([W[r * rb:(r + 1) * rb] for r in rows]), X, 64, N, K)
        assert O.nmse(Ys[:, rows], want) < (1e-10 if N <= 8 else 1e-4), (O.TYPE_NAMES[t], M, N, K)
    if ndev >= 2:
        # a non-main device as the main device
        Ys, _ = ref.mul_mat_split(O.Q4_K, W, X, M, N, K, dev="B2001", main_device=1)
        assert np.array_equal(Ys, Y1[0, 0])


def test_gguf_file_to_device_through_pinned_host_buffer(plugin, tmp_path):
    """SURVEY §8f-4: GGUF file (reference writer) -> reference loader -> device buffer, staged through the backend's pinned host buffer type and
    uploaded with set_tensor_async -> MUL_MAT on the device == the oracle, for hot-path, next and i-quant formats"""
    ref = O.Ref()
    assert ref.load_backend(plugin)
    orc = O.Oracle()
    rng = np.random.default_rng(55)
    for t, M, N, K in [(O.Q4_K, 11008, 1, 4096), (O.Q8_0, 4096, 4, 4096), (O.Q6_K, 1000, 1, 2048), (O.IQ2_XXS, 512, 2, 1024), (O.Q4_0, 4096, 64, 4096)]:
        W = O.random_blocks(t, M * K // orc.blck_size(t), rng)
        X = rng.uniform(-1, 1, N * K).astype(np.float32)
        Y, pinned = ref.gguf_mul_mat(t, W, X, M, N, K, "B2000", tmp_path / "w.gguf")
        assert pinned, "the device must offer a pinned host buffer type"
        rows = rng.choice(M, 64, replace=False)
        rb = orc.row_size(t, K)
        want = orc.mul_mat(t, np.concatenate([W[r * rb:(r + 1) * rb] for r in rows]), X, 64, N, K)
        assert O.nmse(Y[:, rows], want) < (1e-10 if N <= 8 else 1e-4), (O.TYPE_NAMES[t], M, N, K)
