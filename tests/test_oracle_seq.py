"""CPU-only: the f64 references and per-element bounds of oracle/seq.py (ROPE, SSM_CONV, SSM_SCAN, RWKV_WKV6, GATED_LINEAR_ATTN) pinned:
  - each reference against a slow, independent formulation at small shapes (np.longdouble loops; for ROPE the angle recomputed per pair
    as the kernels do and the rotation in long double);
  - every ggml-cpu element (oracle/_ref's one-node probes) within its bound, at model sizes and long prompts reduced to what ggml-cpu runs
    in seconds;
  - a floor: the worst ggml-cpu element must reach FLOOR of its bound, so that no bound becomes vacuous (one 100x too loose fails);
  - the glibc expf / log1pf in use within the 2 ulp the SSM_SCAN bound assumes: on every dt ≤ 20 that three scan cases draw (the
    softplus), and on every f32 argument dt_sp · A of one 8-sequence, d_state 256 case (dA).
Each test prints the worst |y − r| / bound per op and the case where it occurs."""
import ctypes as C

import numpy as np
import pytest

import ggml_b200 as g
from oracle import oracle as O
from oracle import rope as R
from oracle import seq
from oracle import ssm as S
from oracle import wkv as W

# the worst ggml-cpu element measured per op (this file, x86-64 with AVX2): ROPE f32 0.596, f16 0.999, SSM_CONV 0.748, SSM_SCAN y 0.351 /
# states 0.629, RWKV_WKV6 y 0.206 / states 0.993, GATED_LINEAR_ATTN y 0.177 / states 0.993.  FLOOR sits more than 10x below the smallest.
FLOOR = 1e-2
LD = np.longdouble


@pytest.fixture(scope="module", autouse=True)
def need_probes():
    for fam in ("rope", "ssm", "wkv"):
        if not (O.REF_DIR / f"libggml_{fam}_probe.so").exists():
            pytest.skip(f"libggml_{fam}_probe.so not built (oracle/_ref needs the reference tree)")


def _report(op, rows):
    """rows: (case, worst ratio); prints and checks the worst, returns it"""
    case, worst = max(rows, key=lambda r: r[1])
    print(f"{op}: ggml-cpu worst |y - r| / bound {worst:.3g} at {case}")
    assert worst <= 1.0, (op, case, worst)
    assert worst >= FLOOR, (op, case, worst, "bound vacuous")
    return worst


# ------------------------------------------------------------------ cases
POS = (0, -1, -((1 << 24) - 1), 131071, 1 << 20, (1 << 24) - 1, 4095, -4096)


def rope_cases():
    """every mode in f32 and f16, n_dims 0 / partial / ne0, ne0 up to 1024, ne3 = 2 in every mode, the large and negative positions,
    long-context YaRN, llama-3's freq factors (with YaRN on top) and uniform(1, 4) ones"""
    F32, F16 = O.F32, O.F16
    yarn = dict(ext_factor=1.0, freq_scale=1 / 8, attn_factor=1.25, n_ctx_orig=8192)
    return [R.Case(F32, (2, 64, 8, 2), 2, R.ROPE_NORM, positions=POS, seed=1),
            R.Case(F16, (64, 5, 8, 2), 0, R.ROPE_NEOX, positions=POS, seed=2),
            R.Case(F32, (80, 64, 8, 1), 80, R.ROPE_NEOX, positions=POS, seed=3, **yarn),
            R.Case(F16, (96, 12, 8, 2), 64, R.ROPE_NORM, ff=True, positions=POS, seed=4),
            R.Case(F32, (128, 8, 16, 1), 128, R.ROPE_NEOX, ff=True, positions=POS, seed=5, ext_factor=1.0, freq_scale=1 / 32,
                   attn_factor=0.8, n_ctx_orig=8192, freq_base=500000.0, llama3_ff=True),
            R.Case(F16, (256, 4, 8, 2), 256, R.ROPE_NEOX, positions=POS, seed=6, **yarn),
            R.Case(F32, (512, 3, 8, 1), 384, R.ROPE_NORM, positions=POS, seed=7),
            R.Case(F32, (1024, 3, 8, 2), 1024, R.ROPE_NORM, positions=POS, seed=8, **yarn),
            R.Case(F16, (1024, 2, 8, 1), 1024, R.ROPE_NEOX, positions=POS, seed=9),
            R.Case(F32, (128, 12, 8, 2), 128, R.ROPE_MROPE, (24, 20, 20, 0), positions=POS, seed=10, **yarn),
            R.Case(F16, (128, 6, 8, 1), 96, R.ROPE_MROPE, (16, 16, 16, 0), ff=True, positions=POS, seed=11),
            R.Case(F32, (80, 64, 8, 2), 40, R.ROPE_VISION, (10, 10, 0, 0), positions=POS, seed=12),
            R.Case(F16, (80, 16, 8, 1), 40, R.ROPE_VISION, (6, 4, 5, 5), positions=POS, seed=13, **yarn)]


def params_of(case):
    return g.rope_params(case.n_dims, case.mode, case.sections, case.n_ctx_orig, case.freq_base, case.freq_scale, case.ext_factor,
                         case.attn_factor, case.beta_fast, case.beta_slow)


CONV = [S.ConvCase(4, 1000, 512, 4, seed=1), S.ConvCase(4, 5120, 1, 1, seed=2), S.ConvCase(4, 8192, 64, 1, seed=3), S.ConvCase(4, 8192, 1, 4, seed=4)]
SCAN = [S.ScanCase(16, 1000, 2048, 1, bc_rank=48, seed=1), S.ScanCase(16, 1536, 64, 8, bc_rank=160, seed=2),
        S.ScanCase(256, 1000, 1, 8, bc_rank=256, seed=3), S.ScanCase(256, 5120, 4, 1, bc_rank=48, seed=4)]
KEEP = (-8.1, -5.0)             # decays exp(-exp(w)) from 0.9933 to 1 - 3.0e-4
WKV = [W.WkvCase(40, 32, 2048, 1, seed=1, w_range=KEEP), W.WkvCase(64, 32, 512, 1, True, 1.0, seed=2, w_range=KEEP),
       W.WkvCase(80, 40, 16, 3, seed=3), W.WkvCase(128, 40, 1, 8, True, 64 ** -0.5, seed=4), W.WkvCase(200, 32, 4, 3, True, 1.0, seed=5),
       W.WkvCase(256, 64, 1, 3, seed=6), W.WkvCase(256, 32, 2, 1, True, 64 ** -0.5, seed=7)]


# ------------------------------------------------------------------ 1. the references against slow formulations
def test_conv_reference_against_long_double_loops():
    case = S.ConvCase(4, 7, 5, 2, seed=9)
    sx, c = seq.conv_arrays(case)
    r, b = seq.ssm_conv(sx, c)
    for s in range(2):
        for t in range(5):
            for i in range(7):
                want = sum(LD(sx[s, i, t + k]) * LD(c[i, k]) for k in range(4))
                assert abs(LD(r[s, t, i]) - want) <= 1e-6 * b[s, t, i], (s, t, i)


def test_scan_reference_against_long_double_loops():
    case = S.ScanCase(5, 6, 9, 2, bc_rank=3, seed=9)
    s0, x, dt, A, B, Cc = seq.scan_arrays(case)
    y, ey, st, es = seq.ssm_scan(s0, x, dt, A, B, Cc)
    for s in range(2):
        for i in range(6):
            state = [LD(v) for v in s0[s, i]]
            for t in range(9):
                d = LD(dt[s, t, i])
                sp = np.log1p(np.exp(d)) if d <= 20 else d
                state = [state[k] * np.exp(sp * LD(A[i, k])) + LD(B[s, t, k]) * (LD(x[s, t, i]) * sp) for k in range(5)]
                want = sum(state[k] * LD(Cc[s, t, k]) for k in range(5))
                assert abs(LD(y[s, t, i]) - want) <= 1e-6 * ey[s, t, i], (s, t, i)
            for k in range(5):
                assert abs(LD(st[s, i, k]) - state[k]) <= 1e-6 * es[s, i, k], (s, i, k)


@pytest.mark.parametrize("gla", [False, True], ids=["wkv6", "gla"])
def test_wkv_reference_against_long_double_loops(gla):
    case = W.WkvCase(5, 2, 6, 2, gla, 0.37, seed=9)
    args = seq.wkv_args(case, case.sources())
    k, v, a, b, tf, s0 = args[:6]
    y, ey, st, es = seq.wkv(*args)
    for q in range(2):
        for h in range(2):
            state = [[LD(s0[q, h, i, j]) for j in range(5)] for i in range(5)]
            for t in range(q * 6, q * 6 + 6):
                for j in range(5):
                    acc = LD(0)
                    for i in range(5):
                        kv = LD(k[t, h, i]) * LD(v[t, h, j])
                        if gla:
                            state[i][j] = state[i][j] * LD(b[t, h, i]) + kv
                            acc += state[i][j] * (LD(a[t, h, i]) * LD(np.float32(0.37)))
                        else:
                            acc += (kv * LD(tf[h, i]) + state[i][j]) * LD(a[t, h, i])
                            state[i][j] = state[i][j] * LD(b[t, h, i]) + kv
                    assert abs(LD(y[t, h, j]) - acc) <= 1e-6 * ey[t, h, j], (t, h, j)
            for i in range(5):
                for j in range(5):
                    assert abs(LD(st[q, h, i, j]) - state[i][j]) <= 1e-6 * es[q, h, i, j], (q, h, i, j)


def _theta_per_pair(p, pos4, j):
    """the angle of pair j recomputed from the position on its own (the device's rope_theta form), f32 scalars"""
    f = np.float32
    mode, ts = int(p.mode), f(p.theta_scale)
    if not mode & R.ROPE_MROPE:
        t = f(pos4[0])
        for _ in range(j):
            t = f(t * ts)
        return t
    s = [int(p.sections[i]) for i in range(4)]
    bounds = (s[0], s[0] + s[1], s[0] + s[1] + s[2])
    sect = bounds[2] + s[3]
    cur, sector = [f(v) for v in pos4], 0
    for k in range(j + 1):
        if mode == R.ROPE_VISION:
            for w, start in enumerate((0,) + bounds):
                if sector == start:
                    cur[w] = f(pos4[w])
        if k == j:
            return cur[1 if bounds[0] <= sector < bounds[1] else 2 if bounds[1] <= sector < bounds[2] else 3 if sector >= bounds[2] else 0]
        cur = [f(c * ts) for c in cur]
        sector = (sector + 1) % sect


@pytest.mark.parametrize("i", [0, 2, 5, 9, 11])
def test_rope_reference_against_per_pair_angles_and_exact_rotation(i):
    case = rope_cases()[i]
    x, pos, ff = case.inputs()
    p = params_of(case)
    ne0, n_head, n_pos, ne3 = case.ne
    xs = x.reshape(case.ne[::-1])
    r, b = seq.rope(xs, pos, p, ff)
    th = seq.rope_angles(pos, n_pos, p, ff)
    f = np.float32
    ncache = th.shape[1]
    for ip in range(n_pos):
        pos4 = [pos[ip + w * n_pos] if case.multi else (pos[ip] if w == 0 else 0) for w in range(4)]
        for j in range(ncache):
            t = _theta_per_pair(p, pos4, j)
            ext = f(t / f(ff[j] if ff is not None else 1.0))
            want = f(f(p.freq_scale) * ext)
            if case.ext_factor != 0:
                span = f(f(p.corr_dims[1]) - f(p.corr_dims[0]))
                yv = f(f(f(j) - f(p.corr_dims[0])) / max(f(0.001), span))
                mix = f(f(f(1) - min(f(1), max(f(0), yv))) * f(p.ext_factor))
                want = f(f(want * f(f(1) - mix)) + f(ext * mix))
            assert th[ip, j] == want, (ip, j)
    # the rotation in long double, element by element, from the f32 angle
    ms = LD(f(p.mscale))
    nd = case.n_dims
    for i3 in range(ne3):
        for ip in range(n_pos):
            for h in range(min(n_head, 3)):
                row = xs[i3, ip, h]
                for q in range(ne0 // 2):
                    if case.mode == R.ROPE_VISION:
                        e0, e1, slot = q, q + nd, q
                    elif q >= nd // 2:
                        assert r[i3, ip, h, 2 * q] == row[2 * q] and b[i3, ip, h, 2 * q] == 0
                        continue
                    else:
                        e0, e1, slot = (2 * q, 2 * q + 1, q) if case.mode == R.ROPE_NORM else (q, q + nd // 2, q)
                    a = LD(th[ip, slot])
                    cs, sn = np.cos(a) * ms, np.sin(a) * ms
                    w0 = LD(row[e0]) * cs - LD(row[e1]) * sn
                    w1 = LD(row[e0]) * sn + LD(row[e1]) * cs
                    assert abs(LD(r[i3, ip, h, e0]) - w0) <= 1e-6 * b[i3, ip, h, e0]
                    assert abs(LD(r[i3, ip, h, e1]) - w1) <= 1e-6 * b[i3, ip, h, e1]


# ------------------------------------------------------------------ 2. ggml-cpu within the bounds, 3. the floor
def test_rope_cpu_within_bound():
    rows = {O.F32: [], O.F16: []}
    for case in rope_cases():
        x, pos, ff = case.inputs()
        r, b = seq.rope(x.reshape(case.ne[::-1]), pos, params_of(case), ff)
        y = R.probe("CPU", case).reshape(case.ne[::-1])
        rows[case.type].append((str(case), float(seq.ratio(y, r, b).max())))
    _report("ROPE f32", rows[O.F32])
    _report("ROPE f16", rows[O.F16])


def test_ssm_conv_cpu_within_bound():
    rows = []
    for case in CONV:
        r, b = seq.ssm_conv(*seq.conv_arrays(case))
        rows.append((str(case), float(seq.ratio(S.ssm_conv("CPU", case), r, b).max())))
    _report("SSM_CONV", rows)


def test_ssm_scan_cpu_within_bound():
    ys, sts = [], []
    for case in SCAN:
        v = case.views()
        y, st = S.ssm_scan("CPU", case, v)
        ry, ey, rs, es = seq.ssm_scan(*seq.scan_arrays(case, v))
        ys.append((str(case), float(seq.ratio(y, ry, ey).max())))
        sts.append((str(case), float(seq.ratio(st, rs, es).max())))
    _report("SSM_SCAN y", ys)
    _report("SSM_SCAN states", sts)


@pytest.mark.parametrize("gla", [False, True], ids=["wkv6", "gla"])
def test_wkv_cpu_within_bound(gla):
    ys, sts = [], []
    for case in WKV:
        if case.gla != gla:
            case = W.WkvCase(case.S, case.H, case.n_seq_tok, case.n_seqs, gla, W.GLA_SCALES[case.seed % 2] if gla else 1.0, case.seed, case.w_range)
        srcs = case.sources()
        y, st = W.wkv("CPU", case, srcs)
        ry, ey, rs, es = seq.wkv(*seq.wkv_args(case, srcs))
        ys.append((str(case), float(seq.ratio(y, ry, ey).max())))
        sts.append((str(case), float(seq.ratio(st, rs, es).max())))
    name = "GATED_LINEAR_ATTN" if gla else "RWKV_WKV6"
    _report(f"{name} y", ys)
    _report(f"{name} states", sts)


def test_glibc_expf_log1pf_within_the_bounds_ulp_figure():
    m = C.CDLL("libm.so.6")
    for fn in ("expf", "log1pf"):
        getattr(m, fn).restype, getattr(m, fn).argtypes = C.c_float, [C.c_float]
    f32 = np.float32

    def ulps(fn, args, exact):
        got = np.array([fn(float(a)) for a in args], dtype=np.float64)
        return got, float(np.max(np.abs(got - exact) / seq.ulp32(got)))
    # the softplus: every dt <= 20 the cases SCAN[1:] draw
    dts = np.unique(np.concatenate([seq.scan_arrays(c)[2].ravel() for c in SCAN[1:]]))
    dts = dts[dts <= 20.0]
    E, w_exp = ulps(m.expf, dts, np.exp(dts.astype(np.float64)))
    E32 = E.astype(np.float32)
    _, w_log = ulps(m.log1pf, E32, np.log1p(E32.astype(np.float64)))
    # dA: every f32 argument dt_sp * A of SCAN[2] (8 sequences, d_state 256), dt_sp as glibc computes it
    _, _, dt, A, _, _ = seq.scan_arrays(SCAN[2])
    d = dt[:, 0, :]
    sp = np.where(d <= 20.0, np.array([m.log1pf(m.expf(float(v))) for v in d.ravel()], dtype=np.float32).reshape(d.shape), d)
    args = np.unique((sp[:, :, None].astype(f32) * A[None].astype(f32)).astype(f32).ravel())
    _, w_dA = ulps(m.expf, args, np.exp(args.astype(np.float64)))
    print(f"glibc: expf within {w_exp:.3f} ulp on {dts.size} dt values and {w_dA:.3f} ulp on {args.size} dt_sp * A arguments, "
          f"log1pf within {w_log:.3f} ulp (the bound assumes 2)")
    assert max(w_exp, w_dA) <= seq.L_EXP and w_log <= seq.L_LOG1P, (w_exp, w_dA, w_log)


def test_ggml_angle_drift_is_reported():
    d = seq.angle_drift((131071, (1 << 24) - 1))
    print("ggml's f32 ROPE angle chain vs pos * 10000^(-2j/128): " + ", ".join(f"pos {p}: {v:.3g} rad" for p, v in d.items()))
    assert 0 < d[131071] < d[(1 << 24) - 1]
