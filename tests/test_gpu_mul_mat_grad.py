"""GPU: MUL_MAT's backward graph on the device (mul_mat_f_kernel and sum_kernel forward; out_prod_kernel, repeat_back_kernel and the
PERMUTE views backward) against the exact f64 gradient of oracle/grad.py and against ggml-cpu on the same inputs:
  (a) the reference test-backend-ops' f32 x f32 MUL_MAT cases on fixed seeds (tests/test_oracle_mul_mat_grad.py runs them on ggml-cpu):
      every ga element within gamma_P sum |terms| of g, and bit-identical to ggml-cpu's (OUT_PROD is bit-identical on ggml-cpu's SIMD
      body, ne0 = K rounded down to 64, which is all of K = 256; REPEAT_BACK adds in ggml-cpu's order); every gn element within its
      rounding bound (a sample holding the smallest |g| where test-backend-ops skips the case);
  (b) test-backend-ops' MAA check replayed on the same inputs on both backends;
  (c) shapes test-backend-ops never gradient-checks, ga only: M and K up to 4096, N up to 512, bs {3, 2} with nr {2, 2}, each of its
      permutations, and K that is not a multiple of OUT_PROD's 64-element body."""
import numpy as np
import pytest

from oracle import decoder
from oracle import grad as G

import test_oracle_mul_mat_grad as T

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def plugin():
    return decoder.plugin("test-backend-ops", "libggml_grad_probe.so")


def body_mask(case, shape):
    """the elements OUT_PROD computes on ggml-cpu's SIMD body: ggml dim 0 (K, the parents' last numpy axis) below K rounded down to 64"""
    assert case.per[0] == 0
    k = case.k - case.k % 64
    return np.broadcast_to(np.arange(shape[-1]) < k, shape)


@pytest.mark.parametrize("case", G.eval_cases(), ids=str)
def test_device_gradient_within_bounds_and_as_cpu(plugin, case):
    worst_ga, worst_gn, worst_gn_vs_cpu = 0.0, 0.0, 0.0
    for seed in T.SEEDS:
        dev, cpu = T.run("B2000", case, seed), T.run("CPU", case, seed)
        for w in dev["idx"]:
            assert dev[f"ga_ok_{w}"], (case, seed, w)
            assert (dev[f"gn_err_{w}"] <= 1.0).all(), (case, seed, w, dev[f"gn_err_{w}"].max())
            ga, ga_cpu = dev["ga"][w], cpu["ga"][w]
            body = body_mask(case, ga.shape)
            assert np.array_equal(ga.view(np.uint32)[body], ga_cpu.view(np.uint32)[body]), (case, seed, w)
            worst_gn_vs_cpu = max(worst_gn_vs_cpu, float(np.abs(dev["gn"][w].astype(np.float64) - cpu["gn"][w]).max()))
        worst_ga, worst_gn = max(worst_ga, dev["ga_ratio"]), max(worst_gn, dev["gn_ratio"])
    print(f"B2000 {case}: worst |ga - g| / bound {worst_ga:.3g}, |gn - g| / bound {worst_gn:.3g}, ga bit-identical to ggml-cpu, "
          f"max |gn - gn_cpu| {worst_gn_vs_cpu:.3g}")


def test_device_maa_replay(plugin):
    """the MAA check on the same inputs on both backends: the device's failures, like ggml-cpu's, come only from terms at gn's rounding
    floor, and without those terms every MAA is far below the gate"""
    rows = {dev: T.replay(dev, T.CHECKED, T.SEEDS) for dev in ("B2000", "CPU")}
    fails = {dev: len(T.print_replay(dev, r)) for dev, r in rows.items()}
    print(f"MAA failures over {len(rows['CPU'])} checks: B2000 {fails['B2000']}, ggml-cpu {fails['CPU']}")
    T.check_replay(rows["B2000"])


LARGE = [G.GradCase(4096, 512, 4096),
         G.GradCase(1024, 256, 1000, (3, 1), (2, 1)),                            # K % 64 != 0, REPEAT_BACK over 2 batches
         G.GradCase(512, 128, 777, (3, 2), (2, 2)),                              # bs {3, 2}, nr {2, 2}: dB only
         G.GradCase(512, 96, 1000, (3, 1), (2, 1), (0, 2, 1, 3)),
         G.GradCase(512, 96, 1000, (3, 1), (2, 1), (0, 1, 3, 2)),
         G.GradCase(512, 96, 1000, (3, 1), (2, 1), (0, 3, 2, 1)),
         G.GradCase(300, 512, 4096, (2, 3), (1, 1), (0, 3, 2, 1))]


@pytest.mark.parametrize("case", LARGE, ids=str)
def test_large_device_gradient_within_bounds(plugin, case):
    a, b = case.inputs(7)
    ref = G.reference(case, a, b, outputs=False)
    _, ga_a, ga_b, _, _ = G.mul_mat_grad("B2000", case, a, b)
    worst = 0.0
    for ga, g, bound in ((ga_a, ref.g_a, ref.bound_a), (ga_b, ref.g_b, ref.bound_b)):
        if ga is None:
            continue
        err = np.abs(ga.astype(np.float64) - g)
        assert (err <= bound).all(), (case, float((err / bound).max()))
        worst = max(worst, float((err / bound).max()))
    print(f"B2000 {case}: worst |ga - g| / bound {worst:.3g}")
