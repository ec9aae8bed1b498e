"""GPU: the training ops on the device (ops.cu's out_prod_kernel, cross_entropy_loss[_back]_kernel, opt_step_adamw_kernel, argmax_kernel,
count_equal_kernel, sum_kernel, repeat_back_kernel and unary_kernel's STEP) against ggml-cpu and f64:
  (a) the reference's own test-backend-ops on B2000: every case of the nine ops executes and passes; the only ones declined are the
      non-f32 OUT_PROD cases, the I32 / I16 REPEAT_BACK cases, which ggml-cpu itself cannot run, and STEP on non-contiguous views;
  (b) probe parity, B2000 against ggml-cpu, over the host test's grids and at the shapes of a 784-500-10 classifier trained on batches of
      500: OPT_STEP_ADAMW, ARGMAX, COUNT_EQUAL, REPEAT_BACK and STEP bit for bit, OUT_PROD bit for bit on ggml-cpu's SIMD body and within
      NMSE 1e-12 everywhere (also against f64), SUM within 1 ulp, the cross-entropy pair within their bounds of f64;
  (c) one large OUT_PROD (4096 x 4096, K = 2048) against an f64 product;
  (d) the C ABI: error codes, and a captured CUDA graph of OUT_PROD -> CROSS_ENTROPY_LOSS_BACK -> OPT_STEP_ADAMW replayed with new inputs
      and new AdamW hyper-parameters equals eager launches bit for bit."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

from oracle import decoder
from oracle import oracle as O
from oracle import train as TR
from oracle.pool import F32, Source

import test_hostemu_train as H

pytestmark = pytest.mark.gpu
OUT_PROD_NMSE = 1e-12
CE_REL = 1e-5            # CROSS_ENTROPY_LOSS: relative error against f64 (and against ggml-cpu)
CE_BACK_NMSE = 1e-12     # CROSS_ENTROPY_LOSS_BACK against f64, as SOFT_MAX's rows
# test-backend-ops cases per op on B2000 (passed, not supported): the non-f32 OUT_PROD pairs, the I32 / I16 REPEAT_BACK cases and STEP on
# non-contiguous views are the only ones declined
TBO_COUNTS = {"OUT_PROD": (64, 832), "CROSS_ENTROPY_LOSS": (2, 0), "CROSS_ENTROPY_LOSS_BACK": (2, 0), "OPT_STEP_ADAMW": (1, 0), "ARGMAX": (6, 0),
              "COUNT_EQUAL": (1, 0), "SUM": (1, 0), "REPEAT_BACK": (10, 4), "STEP": (2, 2)}
OPS = ("OUT_PROD", "CROSS_ENTROPY_LOSS", "CROSS_ENTROPY_LOSS_BACK", "OPT_STEP_ADAMW", "ARGMAX", "COUNT_EQUAL", "SUM", "REPEAT_BACK", "STEP")


@pytest.fixture(scope="module")
def plugin():
    return decoder.plugin("test-backend-ops", "libggml_train_probe.so")


# ------------------------------------------------------------------ (a) the reference's test-backend-ops
def declined_expected(op, line):
    if op == "OUT_PROD":
        return not ("type_a=f32" in line and "type_b=f32" in line)
    if op == "REPEAT_BACK":
        return "type=i32" in line or "type=i16" in line
    if op == "STEP":                      # the non-contiguous views: like every unary op, STEP takes contiguous f32 only
        return "v=1" in line
    return False


@pytest.mark.parametrize("op", OPS)
def test_reference_test_backend_ops(plugin, op):
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(plugin)
    p = subprocess.run([str(O.REF_DIR / "test-backend-ops"), "test", "-o", op, "-b", "B2000"], env=env, capture_output=True, text=True, timeout=900)
    out = p.stdout + p.stderr
    tail = "\n".join(out.splitlines()[-25:])
    assert p.returncode == 0 and "FAIL" not in out, tail
    cases = [l for l in out.splitlines() if l.strip().startswith(op + "(")]
    declined = [l for l in cases if "not supported" in l]
    ok = [l for l in cases if "OK" in l]
    assert all(declined_expected(op, l) for l in declined), "\n".join(l for l in declined if not declined_expected(op, l))
    assert all(not declined_expected(op, l) for l in ok)
    assert len(ok) + len(declined) == len(cases) and (len(ok), len(declined)) == TBO_COUNTS[op], (len(ok), len(declined), tail)
    m = re.search(r"(\d+)/(\d+) tests passed", out)
    assert m and m.group(1) == m.group(2), tail
    print(f"test-backend-ops {op}: {len(ok)} passed, {len(declined)} not supported")


def grad_run(plugin, op, backend):
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(plugin)
    p = subprocess.run([str(O.REF_DIR / "test-backend-ops"), "grad", "-o", op, "-b", backend], env=env, capture_output=True, text=True, timeout=900)
    out = p.stdout + p.stderr
    return p.returncode, out, sorted(l.strip().split(":")[0] for l in out.splitlines() if "FAIL" in l and l.strip().startswith(op + "("))


@pytest.mark.parametrize("op", ["ADD", "SUB", "MUL", "SCALE", "SUM", "SUM_ROWS", "REPEAT", "CROSS_ENTROPY_LOSS", "UNARY"])
def test_reference_gradients(plugin, op):
    rc, out, failed = grad_run(plugin, op, "B2000")
    assert rc == 0 and "FAIL" not in out, "\n".join(failed[:10] + out.splitlines()[-10:])
    m = re.search(r"(\d+)/(\d+) tests passed", out)
    print(f"test-backend-ops grad {op}: {m.group(0) if m else 'no summary'}")


def test_reference_mul_mat_gradients(plugin):
    """MUL_MAT's gradient (OUT_PROD for both sources, REPEAT_BACK over broadcast batches) on B2000.  An OPEN DEFECT is pinned here, not a
    pass: test-backend-ops draws fresh inputs every run, and on B2000 a run has had up to three f32 x f32 cases (none in some runs) with m = 16, K = 256
    (different ones from run to run, permuted or not) whose finite-difference check exceeds its MAA bound of 1e-4 (1.1e-4 to 6.8e-4 seen),
    where ggml-cpu passed all 3504 cases.  The cause is not isolated.  What is held: every other case passes, and a failure is only that
    MAA check on such a case."""
    rc, out, failed = grad_run(plugin, "MUL_MAT", "B2000")
    lines = [l for l in out.splitlines() if "FAIL" in l and l.strip().startswith("MUL_MAT(")]
    print(f"MUL_MAT grad on B2000: {len(lines)} failing case(s)")
    print("\n".join(lines))
    for l in lines:
        assert "type_a=f32,type_b=f32,m=16," in l and ",k=256," in l and re.search(r"MAA = [0-9.e+-]+ > 0\.000100000 compare failed", l), l


# ------------------------------------------------------------------ (b) probe parity, device vs ggml-cpu
def u32(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def test_adamw_device_is_bit_identical_to_cpu(plugin):
    cases = [(H.adamw_params(*k), H.adamw_inputs(i)) for i, k in enumerate(H.ADAMW_GRID)]
    rng = np.random.default_rng(3)
    # the 784 x 500 weight of the classifier's first layer
    big = tuple(x.reshape(500, 784) for x in H.adamw_inputs(99, 784 * 500))
    cases.append((H.adamw_params(1e-3, 0.9, 0.999, 1e-8, 0.0, 37), big))
    for p, (w, gr, m, v) in cases:
        got, want = TR.opt_step_adamw("B2000", w, gr, m, v, p), TR.opt_step_adamw("CPU", w, gr, m, v, p)
        for a, b in zip(got, want):
            assert np.array_equal(u32(a), u32(b)), p
    print(f"OPT_STEP_ADAMW: {len(cases)} cases bit-identical")


def test_argmax_count_equal_step_device_are_exact(plugin):
    for x in H.argmax_rows():
        assert TR.argmax("B2000", x.reshape(1, -1))[0] == TR.argmax("CPU", x.reshape(1, -1))[0], list(x)
    rng = np.random.default_rng(11)
    for rows, n in ((500, 10), (512, 32000), (10, 5438)):
        x = rng.integers(-50, 50, (rows, n)).astype(np.float32)
        x[rng.integers(0, rows, rows // 3), rng.integers(0, n, rows // 3)] = np.nan
        assert np.array_equal(TR.argmax("B2000", x), TR.argmax("CPU", x)), (rows, n)
    for shape in ((500,), (4, 500), (1000, 3)):
        a = rng.integers(0, 4, shape).astype(np.int32)
        b = rng.integers(0, 4, shape).astype(np.int32)
        assert TR.count_equal("B2000", a, b) == TR.count_equal("CPU", a, b) == int((a == b).sum())
    x = rng.standard_normal((3, 500, 500)).astype(np.float32)
    x.reshape(-1)[:8] = [0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 1e-45, -1e-45]
    assert np.array_equal(u32(TR.step("B2000", x)), u32(TR.step("CPU", x)))


def test_repeat_back_device_is_bit_identical_to_cpu(plugin):
    cases = H.repeat_back_cases()
    # the bias gradients of the classifier: [500, 500] -> [500] and [10, 500] -> [10]
    cases += [(Source(F32, (500, 500), seed=70), (500, 1)), (Source(F32, (10, 500), seed=71), (10, 1))]
    for src, ne in cases:
        parent = H.wide_parent(src)
        assert np.array_equal(u32(TR.repeat_back("B2000", src, ne, parent)), u32(TR.repeat_back("CPU", src, ne, parent))), (src, ne)


def out_prod_f64(sa, sb, pa, pb):
    a64 = pa.astype(np.float64)[..., : sa.ne[1], : sa.ne[0]]
    ne_b, _ = sb.view()
    b64 = np.swapaxes(pb.astype(np.float64), -1, -2) if sb.transpose else pb.astype(np.float64)
    a64 = np.repeat(np.repeat(a64, ne_b[2] // sa.ne[2], axis=1), ne_b[3] // sa.ne[3], axis=0)
    return np.einsum("...km,...kn->...nm", a64, b64)


def test_out_prod_device_against_cpu_and_f64(plugin):
    # the classifier's weight gradients: dW1 = out_prod(x [784, 500], transpose(grad [500, 500])), dW2 = out_prod(h [500, 500], grad^T [10, 500])
    cases = H.out_prod_cases() + [(Source(F32, (784, 500), seed=80), Source(F32, (500, 500), transpose=True, seed=81)),
                                  (Source(F32, (500, 500), seed=82), Source(F32, (500, 10), transpose=True, seed=83)),
                                  (Source(F32, (64, 96, 3, 2), seed=84), Source(F32, (40, 96, 6, 4), seed=85))]
    worst = 0.0
    for sa, sb in cases:
        pa, pb = H.finite_parent(sa), H.finite_parent(sb)
        got, want = TR.out_prod("B2000", sa, sb, pa, pb), TR.out_prod("CPU", sa, sb, pa, pb)
        body = got.shape[-1] - got.shape[-1] % 64
        assert np.array_equal(u32(got[..., :body]), u32(want[..., :body])), (sa, sb)
        if np.any(want):
            e = max(O.nmse(got.reshape(-1), want.reshape(-1)), O.nmse(got.reshape(-1), out_prod_f64(sa, sb, pa, pb).reshape(-1)))
            assert e <= OUT_PROD_NMSE, (sa, sb, e)
            worst = max(worst, e)
        else:
            assert not np.any(got)
    print(f"OUT_PROD B2000: {len(cases)} cases, SIMD body bit-identical to ggml-cpu, worst NMSE {worst:.2e}")


def ce_f64(x, l):
    x64, l64 = x.astype(np.float64), l.astype(np.float64)
    ls = x64 - x64.max(-1, keepdims=True)
    ls = ls - np.log(np.exp(ls).sum(-1, keepdims=True))
    return -(l64 * ls).sum() / (x.size // x.shape[-1]), ls


def ce_inputs(shape, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(shape) * 3).astype(np.float32)
    l = rng.random(shape).astype(np.float32)
    return x, (l / l.sum(-1, keepdims=True)).astype(np.float32)


CE_SHAPES = [(3, 4, 5, 10), (1, 30000), (500, 10), (7, 1), (2, 3, 1000)]


def test_cross_entropy_pair_device_against_f64_and_cpu(plugin):
    worst_rel, worst_back = 0.0, 0.0
    for i, shape in enumerate(CE_SHAPES):
        x, l = ce_inputs(shape, i)
        ref, ls = ce_f64(x, l)
        got, cpu = TR.cross_entropy_loss("B2000", x, l), TR.cross_entropy_loss("CPU", x, l)
        assert got == TR.cross_entropy_loss("B2000", x, l)                          # a fixed order: bit for bit from pass to pass
        rel = max(abs(got - ref), abs(got - cpu)) / max(abs(ref), 1e-30)    # one-class rows: a loss of exactly 0
        assert rel <= CE_REL, (shape, got, cpu, ref)
        worst_rel = max(worst_rel, rel)
        grad = 0.75
        back = TR.cross_entropy_loss_back("B2000", grad, x, l)
        want = (np.exp(ls) - l.astype(np.float64)) * grad / (x.size // x.shape[-1])
        e = O.nmse(back.reshape(-1), want.reshape(-1))
        assert e <= CE_BACK_NMSE, (shape, e)
        worst_back = max(worst_back, e, O.nmse(TR.cross_entropy_loss_back("CPU", grad, x, l).reshape(-1), want.reshape(-1)))
    print(f"CROSS_ENTROPY_LOSS: worst relative error {worst_rel:.2e}; CROSS_ENTROPY_LOSS_BACK: worst NMSE {worst_back:.2e} (ggml-cpu's included)")


def test_sum_device_within_one_ulp(plugin):
    rng = np.random.default_rng(5)
    for shape, parent in (((10, 5, 4, 3), None), ((1 << 20,), None), ((7, 33), (9, 40)), ((500, 10), None), ((3, 1), None)):
        src = Source(F32, shape, parent_ne=parent, seed=len(shape))
        x = (rng.standard_normal(src.parent_ne[::-1]) * 10.0 ** rng.integers(-3, 4, src.parent_ne[::-1])).astype(np.float32)
        got, want = TR.sum_("B2000", src, x), TR.sum_("CPU", src, x)
        assert abs(float(got) - float(want)) <= np.spacing(np.float32(abs(want))), (shape, got, want)


def test_what_ggml_cpu_reads_differently_is_declined(plugin):
    # COUNT_EQUAL over more than a matrix: ggml-cpu's row walk names other rows
    a = np.zeros((3, 5, 4), dtype=np.int32)
    assert TR.count_equal("B2000", a, a, raw=True) == -2


# ------------------------------------------------------------------ (c) one large OUT_PROD
def test_large_out_prod_against_f64():
    import torch
    import ggml_b200 as g
    gen = torch.Generator(device="cuda").manual_seed(0)
    a = torch.rand((2048, 4096), device="cuda", generator=gen) * 2 - 1            # [K, M]
    b = (torch.rand((4096, 2048), device="cuda", generator=gen) * 2 - 1).t()      # [K, N], transposed like the gradient
    y = g.op_out_prod(a, b)
    ref = a.double().t() @ b.double()                                            # [M, N]
    e = (((y.double().t() - ref) ** 2).sum() / (ref ** 2).sum()).item()
    assert e <= OUT_PROD_NMSE, e
    print(f"OUT_PROD 4096 x 4096, K = 2048: NMSE {e:.2e} against f64")


# ------------------------------------------------------------------ (d) the C ABI
def test_c_abi_error_codes():
    import torch
    import ggml_b200 as g
    L = g.lib()
    TD = C.POINTER(g.TensorDesc)
    D = g.strided_desc
    z = lambda *shape, dt=torch.float32: torch.zeros(shape, dtype=dt, device="cuda")
    L.ggml_b200_op_out_prod.argtypes = [TD] * 3 + [C.c_void_p]
    op = lambda a, b, d: L.ggml_b200_op_out_prod(C.byref(D(a)), C.byref(D(b)), C.byref(D(d)), None)
    assert op(z(7, 16), z(7, 5), z(5, 16)) == 0 and op(z(7, 16), z(6, 5), z(5, 16)) == -2 and op(z(7, 16).half(), z(7, 5), z(5, 16)) == -1
    assert op(z(16, 7).t(), z(7, 5), z(5, 16)) == -1 and op(z(7, 16), z(5, 7).t(), z(5, 16)) == 0
    L.ggml_b200_op_opt_step_adamw.argtypes = [TD] * 5 + [C.c_void_p]
    ad = lambda w, p: L.ggml_b200_op_opt_step_adamw(*(C.byref(D(t)) for t in (w, w, w, w, p)), None)
    assert ad(z(10, 5), z(7)) == 0 and ad(z(10, 5), z(6)) == -2 and ad(z(10, 6)[:, :5], z(7)) == -1
    L.ggml_b200_op_count_equal.argtypes = [TD] * 3 + [C.c_void_p]
    ce = lambda a, d: L.ggml_b200_op_count_equal(C.byref(D(a)), C.byref(D(a)), C.byref(D(d)), None)
    i32 = torch.int32
    assert ce(z(5, 4, dt=i32), z(1, dt=torch.int64)) == 0 and ce(z(5, 4, dt=i32), z(1, dt=i32)) == -1 and ce(z(3, 5, 4, dt=i32), z(1, dt=torch.int64)) == -1
    L.ggml_b200_op_argmax.argtypes = [TD] * 2 + [C.c_void_p]
    am = lambda x, d: L.ggml_b200_op_argmax(C.byref(D(x)), C.byref(D(d)), None)
    assert am(z(5, 100), z(5, dt=i32)) == 0 and am(z(5, 100), z(4, dt=i32)) == -2 and am(z(5, 100), z(5)) == -1
    L.ggml_b200_op_repeat_back.argtypes = [TD] * 2 + [C.c_void_p]
    rb = lambda x, d: L.ggml_b200_op_repeat_back(C.byref(D(x)), C.byref(D(d)), None)
    assert rb(z(4, 6), z(2, 3)) == 0 and rb(z(4, 6), z(3, 3)) == -2 and rb(z(4, 6, dt=i32), z(2, 3, dt=i32)) == -1
    torch.cuda.synchronize()


def test_c_abi_cuda_graph_replay_matches_eager():
    import torch
    import ggml_b200 as g
    torch.cuda.set_device(0)
    x = torch.zeros((500, 784), device="cuda")            # [batch, in]
    dlog = torch.zeros((500, 10), device="cuda")           # logits of the batch
    labels = torch.zeros((500, 10), device="cuda")
    w = torch.zeros((10, 784), device="cuda")              # a weight [out, in] and its moments
    m, v = torch.zeros_like(w), torch.zeros_like(w)
    params = torch.zeros(7, device="cuda")
    one = torch.ones(1, device="cuda")

    def chain():
        gl = g.op_cross_entropy_loss_back(one, dlog, labels)               # [500, 10]
        gw = g.op_out_prod(x, gl)                                           # [10, 784] = sum over the batch of gl^T x
        g.op_opt_step_adamw(w, gw, m, v, params)
        return gl, gw
    state = lambda: [t.clone() for t in (w, m, v)]
    init = state()
    chain()
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        captured = chain()
    rng = np.random.default_rng(71)
    for it in range(1, 4):
        x.copy_(torch.from_numpy(rng.standard_normal(x.shape).astype(np.float32)))
        dlog.copy_(torch.from_numpy(rng.standard_normal(dlog.shape).astype(np.float32)))
        labels.copy_(torch.nn.functional.one_hot(torch.from_numpy(rng.integers(0, 10, 500)), 10).float())
        params.copy_(torch.from_numpy(H.adamw_params(10.0 ** -it, 0.9, 0.999, 1e-8, 0.01 * it, it)))
        for t, s in zip((w, m, v), init):
            t.copy_(s)
        graph.replay()
        torch.cuda.synchronize()
        after_graph = [c.clone() for c in captured] + state()
        for t, s in zip((w, m, v), init):
            t.copy_(s)
        eager = list(chain()) + state()
        torch.cuda.synchronize()
        for a, b in zip(after_graph, eager):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        init = state()


# ------------------------------------------------------------------ (e) training through ggml_opt (oracle/train_graph.cpp)
TRAINER = O.REF_DIR / "train-graph"
TRAIN_CALLS = 20                       # forward_backward calls: 10 optimizer steps at opt_period 2
# free-running bounds against ggml-cpu, about 10 x the worst measured: the loss of every call (relative) and the final weights (NMSE)
# (measured: fc 9.8e-7 and 1.9e-14, mse 0 and 1.4e-14)
LOSS_REL = {"fc": 1e-5, "mse": 1e-5}
WEIGHTS_NMSE = {"fc": 2e-13, "mse": 2e-13}


def train(preset, device, out, env_extra=None):
    import ggml_b200
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(ggml_b200.BACKEND_SO)
    env.update(env_extra or {})
    p = subprocess.run([str(TRAINER), preset, "run", device, str(TRAIN_CALLS), str(out)], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, (p.stdout + p.stderr)[-3000:]
    graphs, losses, acc, ms = {}, [], None, None
    for l in p.stdout.splitlines():
        f = l.split()
        if f[0] == "graph":
            graphs[f[1]] = dict(n_splits=int(f[3]), cpu_nodes=int(f[5]), ops=f[6:])
        elif f[0] == "loss":
            losses.append(float(f[2]))
        elif f[0] == "accuracy":
            acc = float(f[1])
        elif f[0] == "ms_per_call":
            ms = float(f[1])
    return dict(graphs=graphs, losses=np.array(losses), accuracy=acc, ms=ms, weights=np.fromfile(out, dtype=np.float32), stdout=p.stdout,
                stderr=p.stderr)


@pytest.mark.parametrize("preset", ["fc", "mse"])
def test_trainer_runs_on_the_device_in_one_split(plugin, preset, tmp_path):
    dev = train(preset, "B2000", tmp_path / "dev.bin")
    # gb_grad and gb_opt: forward, backward and the OPT_STEP_ADAMW nodes (whose hyper-parameters sit in ggml_opt's host buffer) all on B2000
    assert dev["graphs"] == {"grad": dict(n_splits=1, cpu_nodes=0, ops=[]), "opt": dict(n_splits=1, cpu_nodes=0, ops=[])}, dev["graphs"]
    again = train(preset, "B2000", tmp_path / "again.bin")
    no_fusion = train(preset, "B2000", tmp_path / "nofuse.bin", {"GGML_B200_DISABLE_FUSION": "1"})
    no_graphs = train(preset, "B2000", tmp_path / "nograph.bin", {"GGML_B200_DISABLE_GRAPHS": "1"})
    for other in (again, no_fusion, no_graphs):
        assert np.array_equal(other["losses"], dev["losses"]) and np.array_equal(other["weights"].view(np.uint32), dev["weights"].view(np.uint32))
    profiled = train(preset, "B2000", tmp_path / "prof.bin", {"GGML_B200_PROFILE": "1"})
    print(f"{preset}: graph_compute modes with opt_period 2:")
    print("\n".join(l for l in profiled["stderr"].splitlines() if "profile" in l))


@pytest.mark.parametrize("preset", ["fc", "mse"])
def test_trainer_free_running_against_cpu(plugin, preset, tmp_path):
    dev, cpu = train(preset, "B2000", tmp_path / "dev.bin"), train(preset, "CPU", tmp_path / "cpu.bin")
    rel = np.abs(dev["losses"] - cpu["losses"]) / np.abs(cpu["losses"])
    e_w = O.nmse(dev["weights"].astype(np.float64), cpu["weights"].astype(np.float64))
    print(f"{preset}: losses {np.round(dev['losses'], 5).tolist()}")
    print(f"{preset}: worst loss relative difference {rel.max():.2e}, final weights NMSE {e_w:.2e}, accuracy of the last batch "
          f"{dev['accuracy']:.3f} (ggml-cpu {cpu['accuracy']:.3f}); ms per forward_backward call B2000 {dev['ms']:.3f}, ggml-cpu 8 threads {cpu['ms']:.3f}")
    assert dev["losses"][-1] < 0.5 * dev["losses"][0]
    assert rel.max() <= LOSS_REL[preset] and e_w <= WEIGHTS_NMSE[preset], (rel.max(), e_w)
