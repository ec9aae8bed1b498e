"""CPU-only: MUL_MAT's gradient on ggml-cpu (oracle/_ref/libggml_grad_probe.so's probe_mul_mat_grad) against the exact f64 gradient of
oracle/grad.py, over the reference test-backend-ops' f32 x f32 MUL_MAT cases (plain, broadcast and permuted) on fixed seeds:
  - the reference itself against a brute-force f64 perturbation of the loss on small cases of every layout;
  - every element of the backward graph's gradient ga within gamma_P sum |terms| of the exact gradient g;
  - test-backend-ops' numerical gradient gn within its rounding bound, on every element for the cases test-backend-ops checks (at most
    GRAD_NMAX gradient elements) and on a sample holding the smallest |g| for the others;
  - the MAA check replayed on the same inputs: what fails is explained by elements whose |g| is at gn's rounding floor.
tests/test_gpu_mul_mat_grad.py runs the same inputs on the device."""
import numpy as np
import pytest

from oracle import grad as G
from oracle import oracle as O

SEEDS = (0, 1, 2, 3)
SAMPLE = 256                  # gn elements per parameter for the cases test-backend-ops does not check
# gn's rounding floor: |gn - ga| stays within GN_NOISE everywhere (measured on ggml-cpu over 20 seeds: 1.64e-4; the gate is about 10x),
# so an element whose |g| is far below G_FLOOR adds a term of order 1 or more to the MAA, where the gate is 1e-4 for the mean.  Over the
# elements with |g| >= G_FLOOR every replayed MAA passes test-backend-ops' own gate (measured on ggml-cpu over 20 seeds: at most 3.8e-5).
GN_NOISE = 2e-3
G_FLOOR = 0.1
MAA_REST = G.MAA_MAX


@pytest.fixture(scope="module", autouse=True)
def need_probe():
    if not (O.REF_DIR / "libggml_grad_probe.so").exists():
        pytest.skip("libggml_grad_probe.so not built (oracle/_ref needs the reference tree)")


def _brute_force(case, a, b):
    A, B = G._logical(case, a), G._logical(case, b)
    Ab = np.repeat(np.repeat(A, case.nr[0], 2), case.nr[1], 3)
    return float(np.einsum("kmij,knij->", Ab, B))


SMALL = [G.GradCase(3, 2, 4, (2, 1), (2, 1)), G.GradCase(3, 4, 5, (3, 2), (2, 2)), G.GradCase(3, 2, 5, (2, 3), (1, 1), (0, 2, 1, 3)),
         G.GradCase(3, 2, 5, (2, 1), (2, 1), (0, 1, 3, 2)), G.GradCase(3, 2, 5, (2, 3), (1, 1), (0, 3, 2, 1))]


@pytest.mark.parametrize("case", SMALL, ids=str)
def test_reference_is_the_derivative_of_the_loss(case):
    """L is bilinear: L(x + e_i) - L(x) in f64 is the exact gradient at i, for every element of each parameter, in the parents' layouts"""
    a, b = case.inputs(1)
    ref = G.reference(case, a, b)
    l0 = _brute_force(case, a, b)
    assert abs(l0 - ref.loss) <= 1e-12 * max(1.0, abs(l0))
    for which, x, g in (("a", a, ref.g_a), ("b", b, ref.g_b)):
        if g is None:
            continue
        for i in range(x.size):
            xp = x.astype(np.float64).reshape(-1).copy()
            xp[i] += 1.0
            xp = xp.reshape(x.shape)
            d = (_brute_force(case, xp, b) if which == "a" else _brute_force(case, a, xp)) - l0
            assert abs(d - g.reshape(-1)[i]) <= 1e-12, (which, i)


def run(dev, case, seed):
    """the probe on `dev` with every gn (cases test-backend-ops checks) or a sample (the others), and the per-element ratios to the bounds"""
    a, b = case.inputs(seed)
    ref = G.reference(case, a, b)
    full = case.ngrads() <= G.GRAD_NMAX
    idx = {w: (np.arange(x.size, dtype=np.int64) if full else G.sample(g, SAMPLE, seed)) for w, x, g in (("a", a, ref.g_a), ("b", b, ref.g_b))
           if g is not None}
    loss, ga_a, ga_b, gn_a, gn_b = G.mul_mat_grad(dev, case, a, b, idx.get("a"), idx.get("b"))
    out = dict(loss=loss, ref=ref, idx=idx, ga={"a": ga_a, "b": ga_b}, gn={"a": gn_a, "b": gn_b}, full=full, ga_ratio=0.0, gn_ratio=0.0, maa={})
    for w, x in (("a", a), ("b", b)):
        if w not in idx:
            continue
        g, bound = (ref.g_a, ref.bound_a) if w == "a" else (ref.g_b, ref.bound_b)
        ga = out["ga"][w]
        out["ga_ratio"] = max(out["ga_ratio"], float((np.abs(ga.astype(np.float64) - g) / np.maximum(bound, 1e-300)).max()))
        gb_, gi = G.gn_bound(case, ref, w, idx[w], x.reshape(-1)[idx[w]])
        out[f"gn_err_{w}"] = np.abs(out["gn"][w].astype(np.float64) - gi) / gb_
        out["gn_ratio"] = max(out["gn_ratio"], float(out[f"gn_err_{w}"].max()))
        out[f"ga_ok_{w}"] = bool((np.abs(ga.astype(np.float64) - g) <= bound).all())
        if full:
            out["maa"][w] = G.maa(out["gn"][w], ga.reshape(-1))
    return out


@pytest.mark.parametrize("case", G.eval_cases(), ids=str)
def test_cpu_gradient_within_bounds(case):
    worst_ga, worst_gn = 0.0, 0.0
    for seed in SEEDS:
        r = run("CPU", case, seed)
        for w in r["idx"]:
            assert r[f"ga_ok_{w}"], (case, seed, w)
            assert (r[f"gn_err_{w}"] <= 1.0).all(), (case, seed, w, r[f"gn_err_{w}"].max())
        worst_ga, worst_gn = max(worst_ga, r["ga_ratio"]), max(worst_gn, r["gn_ratio"])
    print(f"CPU {case}: worst |ga - g| / bound {worst_ga:.3g}, |gn - g| / bound {worst_gn:.3g} ({'every' if r['full'] else SAMPLE} gn)")


def replay(dev, cases, seeds):
    """test-backend-ops' MAA check on the same inputs: per (case, seed, parameter), the MAA, the worst term and |g| there, the number of
    elements with |g| < G_FLOOR, the MAA over the others, and the largest |gn - ga|"""
    rows = []
    for case in cases:
        for seed in seeds:
            r = run(dev, case, seed)
            for w, m in r["maa"].items():
                gn, ga = r["gn"][w], r["ga"][w].reshape(-1)
                terms = G.maa_terms(gn, ga)
                g = (r["ref"].g_a if w == "a" else r["ref"].g_b).reshape(-1)
                i = int(np.nanargmax(terms))
                keep = np.abs(g) >= G_FLOOR
                rows.append(dict(case=case, seed=seed, param=w, maa=m, worst_term=float(terms[i]), g_at_worst=float(g[i]), n_floor=int((~keep).sum()),
                                 rest=float(terms[keep].sum() / keep.sum()), noise=float(np.abs(gn.astype(np.float64) - ga).max())))
    return rows


def print_replay(dev, rows):
    fails = [r for r in rows if r["maa"] > G.MAA_MAX]
    print(f"{dev}: MAA replay of {len(rows)} (case, seed, parameter) checks: {len(fails)} over {G.MAA_MAX}")
    for r in fails:
        print(f"  {r['case']} seed {r['seed']} d{r['param'].upper()}: MAA {r['maa']:.3g}, worst term {r['worst_term']:.3g} at |g| = "
              f"{abs(r['g_at_worst']):.3g}, {r['n_floor']} element(s) with |g| < {G_FLOOR}, MAA over the others {r['rest']:.3g}")
    print(f"{dev}: worst MAA over |g| >= {G_FLOOR}: {max(r['rest'] for r in rows):.3g}; worst |gn - ga|: {max(r['noise'] for r in rows):.3g}")
    return fails


def check_replay(rows):
    for r in rows:
        where = (r["case"], r["seed"], r["param"])
        assert r["noise"] <= GN_NOISE and r["rest"] <= MAA_REST, (where, r["noise"], r["rest"])
        if r["maa"] > G.MAA_MAX:                                           # a failure needs a term no element above the floor can give
            assert abs(r["g_at_worst"]) < G_FLOOR and r["worst_term"] * r["n_floor"] > 0, where


CHECKED = [c for c in G.eval_cases() if c.ngrads() <= G.GRAD_NMAX]


def test_cpu_maa_replay():
    """ggml-cpu fails test-backend-ops' MAA check on fixed inputs too, and only through elements whose |g| is at gn's rounding floor:
    |gn - ga| stays within GN_NOISE everywhere, and over the elements with |g| >= G_FLOOR every MAA is far below the gate."""
    rows = replay("CPU", CHECKED, SEEDS)
    print_replay("CPU", rows)
    check_replay(rows)
