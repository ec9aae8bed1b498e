"""GPU: GGML_OP_ROPE on the device (ops.cu rope_kernel behind ggml_b200_op_rope and the plug-in).

  * the reference's own test-backend-ops runs every ROPE case (f32 / f16; llama, neox, stablelm, phi-2, qwen2vl m-rope and ViT shapes;
    strided views, freq factors, YaRN) on B2000 against ggml-cpu: all executed, none declined, none failing;
  * one-node ROPE graphs through the reference's graph API (oracle/rope_probe.cpp) on B2000 and on ggml-cpu agree over the grid of
    tests/test_hostemu_rope.py plus in-place cases: f32 to NMSE <= 1e-12, f16 to one f16 ulp per element (only the device sinf / cosf
    differ from glibc's);
  * the C ABI directly: positions are read on the device (a captured CUDA graph rotates by the positions set before each replay), and
    what the CPU backend asserts comes back as an error code."""
import re
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from oracle import rope as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def plugin():
    import ggml_b200
    if not ggml_b200.BACKEND_SO.exists():
        pytest.fail(f"{ggml_b200.BACKEND_SO} missing: run __graft_entry__.build() where the ggml headers are available")
    if not (O.REF_DIR / "test-backend-ops").exists():
        pytest.fail("oracle/_ref/test-backend-ops missing (built by oracle/Makefile in the build container)")
    return ggml_b200.BACKEND_SO


def test_reference_test_backend_ops_rope(plugin):
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(plugin)
    p = subprocess.run([str(O.REF_DIR / "test-backend-ops"), "test", "-o", "ROPE", "-b", "B2000"], env=env, capture_output=True, text=True, timeout=900)
    out = p.stdout + p.stderr
    tail = "\n".join(out.splitlines()[-25:])
    assert p.returncode == 0 and "FAIL" not in out, tail
    cases = [l for l in out.splitlines() if l.strip().startswith("ROPE(")]
    declined = [l for l in cases if "not supported" in l]
    assert not declined, "\n".join(declined[:10])
    ok = [l for l in cases if "OK" in l]
    assert len(ok) == len(cases) and len(ok) >= 100, (len(ok), len(cases), tail)
    for shape in ("ne_a=[128,32,2,1]", "ne_a=[80,32,2,1],n_dims=20", "mode=8", "mode=24", "v=1", "ff=1", "ef=0.746500"):
        assert any(shape in l for l in ok), f"no executed ROPE case with {shape}"
    m = re.search(r"(\d+)/(\d+) tests passed", out)
    assert m and m.group(1) == m.group(2), tail


def test_rope_device_matches_cpu_over_the_grid(plugin):
    ref = O.Ref()
    assert ref.load_backend(plugin)
    worst, flips = 0.0, 0
    cases = R.grid(inplace=True)
    for case in cases:
        got = R.probe("B2000", case)
        want = R.probe("CPU", case)
        if case.type == O.F32:
            err = O.nmse(got.astype(np.float64), want.astype(np.float64))
            worst = max(worst, err)
            assert err <= 1e-12, (str(case), err)
        else:
            # f16 results: a few-ulp sinf / cosf difference can move a value across an f16 rounding boundary (one such element alone is
            # NMSE ~1e-11), so the f16 gate is per element: equal, or one f16 ulp apart
            gi, wi = got.view(np.int16).astype(np.int32), want.view(np.int16).astype(np.int32)
            apart = np.abs(got.astype(np.float64) - want.astype(np.float64))
            ulp = np.spacing(np.maximum(np.abs(got), np.abs(want)).astype(np.float16)).astype(np.float64)
            assert np.all(apart <= ulp), (str(case), float(np.max(apart / ulp)))
            flips += int(np.count_nonzero(gi != wi))
    print(f"ROPE B2000 vs ggml-cpu: {len(cases)} cases, worst f32 NMSE {worst:.2e}, f16 elements one ulp apart: {flips}")


def test_rope_c_abi_positions_are_read_at_replay():
    import torch
    import ggml_b200 as g
    torch.cuda.set_device(0)
    rng = np.random.default_rng(7)
    x = torch.from_numpy(rng.uniform(-1, 1, (1, 9, 16, 128)).astype(np.float32)).cuda()      # [ne3, n_pos, n_head, head]
    pos = torch.zeros(9, dtype=torch.int32, device="cuda")
    p = g.rope_params(128, g.ROPE_NEOX, n_ctx_orig=4096, freq_scale=0.5, ext_factor=1.0)
    g.op_rope(x, pos, p)                                                                      # lazy per-device set-up outside the capture
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        y = g.op_rope(x, pos, p)
    for start in (0, 100, 4000):
        pos.copy_(torch.arange(start, start + 9, dtype=torch.int32))
        graph.replay()
        direct = g.op_rope(x, pos, p)
        torch.cuda.synchronize()
        assert torch.equal(y, direct), start
    assert not torch.equal(y, x)                                                              # the last replay rotated by positions 4000..4008


def test_rope_c_abi_rejects_what_the_cpu_asserts():
    import torch
    import ggml_b200 as g
    x = torch.zeros((1, 2, 4, 64), dtype=torch.float32, device="cuda")
    pos = torch.zeros(2, dtype=torch.int32, device="cuda")
    bad = [g.rope_params(63), g.rope_params(66), g.rope_params(64, 5), g.rope_params(64, g.ROPE_VISION), g.rope_params(64, g.ROPE_MROPE)]
    for p in bad:
        with pytest.raises(g.B200Error):
            g.op_rope(x, pos, p)
    with pytest.raises(g.B200Error):                                                           # MROPE needs four positions per token
        g.op_rope(x, pos, g.rope_params(64, g.ROPE_MROPE, sections=(16, 8, 8, 0)))
    with pytest.raises(g.B200Error):                                                           # freq factors: at least n_dims/2
        g.op_rope(x, pos, g.rope_params(64), freq_factors=torch.ones(31, device="cuda"))
