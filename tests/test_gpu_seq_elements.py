"""GPU: the sequence ops' kernels (ops.cu rope_kernel, ssm_conv_kernel, ssm_scan_kernel, wkv_kernel<GLA>, concat_kernel in the conv-state
hand-off) checked on every output element against the f64 references of oracle/seq.py, through poisoned outputs, chunked prompts and
dependent launches.

Every launch goes through the C ABI into the middle of a NaN-filled buffer between NaN-sentinel guard bands: every element must be
written, lie within its bound (|y − r| ≤ bound), and the guards must stay intact; a relaunch into zeros must give the same bits.  Each case
is also compared with ggml-cpu (oracle/_ref's one-node probes) on the same inputs: SSM_CONV bit-identical, WKV bit-identical at S % 16 == 0
(ggml-cpu's vector path in every column) and within the sum of both bounds elsewhere, SSM_SCAN element by element within the sum of both
bounds (the max ulp distance is printed), ROPE f16 within one f16 ulp (or, across zero, both within their bound) and f32 within the sum
of both bounds.  torch.profiler reads back that each case ran its op's kernel, and that each chunk chain and graph replay launches its
op's kernels and nothing else, in a Python process of its own (ran()).

Shapes: each axis of ROPE (ne0 2 .. 1024, n_dims 0 / partial / ne0, a partial last block of heads, a 4096-position prefill, ne3 > 1, all
four modes in f32 and f16, positions 0, ±(2^24 − 1), 131071, 2^20, long-context YaRN and freq factors, the f16 K-shift in place on a strided
cache view), SSM_CONV (d_inner 1000 / 5120 / 8192, n_t 1 / 512, n_s 1 / 4), SSM_SCAN (d_inner 1000 / 1536 / 5120 / 8192, d_state 16 / 256,
n_t 1 / 2048, n_s 1 / 8, B and C strided views of x_db with dt_rank 48 / 160 / 256) and WKV (S 40 / 64 / 80 / 128 / 200 / 256, H 32 / 40 /
64, 1 or 2048 tokens per sequence, 1 / 3 / 8 sequences, decays up to 1 − 3e-4, both GLA scales) appears in at least one case; long prompts
go with small states, the largest states with short prompts.

Chunk invariance: a 2048-token prompt in one call, and as chunks of 1, of 7 and of 512 tokens, each call's final state fed back as the
next call's s0 (for the conv: op_concat of the last d_conv − 1 columns, as the Mamba layer does): y and the final state bit-identical.
Dependent launches: the chunk-7 chain enqueued with no synchronisation (PDL on) equals the chain synchronised after every launch, and one
chunk step captured as a CUDA graph and replayed over the 512-token chunks gives the same bits.

The f64 references and ggml-cpu take about two minutes of CPU time for the whole file.

The per-element gate is the bound itself (ratio ≤ 1).  Worst |y − r| / bound measured on an NVIDIA H100 80GB HBM3 at its 700 W power limit:
ROPE 1.00 to three digits (the f16 prefill: the store's half ulp dominates), SSM_CONV 0.792, SSM_SCAN y 0.351 / states 0.653, WKV y 0.215 /
states 0.993.  Against ggml-cpu: SSM_CONV bit-identical, WKV bit-identical at S % 16 == 0, ROPE f16 11 elements more than one ulp apart
(near zero, both sides within their bound)."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import rope as R
from oracle import seq
from oracle import ssm as S
from oracle import wkv as W
import test_oracle_seq as T

pytestmark = pytest.mark.gpu

GUARD = 1024
SENTINEL32, SENTINEL16 = 0x7FC0DEAD, 0x7E5A      # NaNs no kernel writes
CHUNKS = (1, 7, 512)
N_LONG = 2048


@pytest.fixture(scope="module")
def g():
    import torch
    import ggml_b200
    assert torch.cuda.is_available(), "these tests need an H100"
    torch.cuda.set_device(0)
    return ggml_b200


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Poisoned:
    """n elements of dtype (torch.float32 / float16) between NaN-sentinel guard bands, filled with NaN"""

    def __init__(self, n, dtype):
        import torch
        it, sent = (torch.int32, SENTINEL32) if dtype == torch.float32 else (torch.int16, SENTINEL16)
        self.buf = torch.full((n + 2 * GUARD,), sent, dtype=it, device="cuda")
        self.sent, self.n = sent, n
        self.y = self.buf[GUARD:GUARD + n].view(dtype)
        self.y.fill_(float("nan"))

    def guards_ok(self):
        return bool((self.buf[:GUARD] == self.sent).all()) and bool((self.buf[GUARD + self.n:] == self.sent).all())


def kernels_of(fn):
    """the CUDA kernel names fn launches (torch.profiler: its raw activity records and its event tree)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    cuda = torch.autograd.DeviceType.CUDA
    raw = {e.name() for e in prof.profiler.kineto_results.events() if e.device_type() == cuda}
    return raw | {e.name for e in prof.events() if e.device_type == cuda}


def packed(t):
    """a packed copy of t (a slice whose leading extent is 1 keeps its parent's stride there, which the ops' packing checks refuse)"""
    import torch
    return torch.empty(t.shape, dtype=t.dtype, device=t.device).copy_(t)


def ran(family: str, kernels, only: bool = False) -> None:
    """every case of `family` ran each of `kernels` (name substrings), and with `only` no other kernel, read back with torch.profiler in a
    new Python process (_names_of).
    On these shared H100 machines the profiler has been seen to record none of a session's kernels, for a whole process, from the first
    session or only after a few; so the read-back runs in a process of its own, at most three times."""
    import json
    import subprocess
    import sys
    from pathlib import Path
    here = Path(__file__).resolve().parent
    code = (f"import sys; sys.path[:0] = [{str(here)!r}, {str(here.parent)!r}]; import json, test_gpu_seq_elements as t; "
            f"print(json.dumps(t._names_of({family!r})))")
    for _ in range(3):
        p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=str(here.parent))
        assert p.returncode == 0, p.stderr[-2000:]
        per_case = json.loads(p.stdout.strip().splitlines()[-1])
        missing = [(i, names) for i, names in enumerate(per_case)
                   if not all(any(k in n for n in names) for k in kernels) or (only and not all(any(k in n for k in kernels) for n in names))]
        if not missing:
            return
    raise AssertionError((family, kernels, missing[:3]))


def _names_of(family: str) -> list:
    """the kernel names of each case of `family`, one profiler session per case (run by ran() in a new process)"""
    import torch
    import ggml_b200 as g
    torch.cuda.set_device(0)
    out = []
    if family == "rope":
        for case in rope_gpu_cases():
            x, pos, ff = case.inputs()
            X, P, FF = dev(x.reshape(case.ne[::-1])), dev(pos), (dev(ff) if ff is not None else None)
            p = T.params_of(case)
            out.append(sorted(kernels_of(lambda: g.op_rope(X, P, p, FF))))
    elif family == "kshift":
        cache = torch.zeros((512, 8, 128), dtype=torch.float16, device="cuda")
        P = torch.zeros(384, dtype=torch.int32, device="cuda")
        out.append(sorted(kernels_of(lambda: g.op_rope(cache[64:448, 1:7, :].unsqueeze(0), P, g.rope_params(128, g.ROPE_NEOX), inplace=True))))
    elif family == "conv":
        for case in CONV:
            SX, Cw = (dev(a) for a in seq.conv_arrays(case))
            out.append(sorted(kernels_of(lambda: g.op_ssm_conv(SX, Cw))))
    elif family == "scan":
        for case in SCAN:
            _, s0, x, dt, A, xdb = scan_inputs(case)
            D = [dev(a) for a in (s0, x, dt, A, xdb)]
            out.append(sorted(kernels_of(lambda: scan_launch(g, *D, case.bc_rank, case.d_state))))
    elif family == "wkv":
        for case in WKV:
            D = [dev(a) for a in case.sources()]
            out.append(sorted(kernels_of(lambda: wkv_launch(g, case, D))))
    elif family == "scan_chain":                      # the first chunks of the chunk-7 chain, back to back
        steps = ScanChain(g).steps(7)[0][:3]
        out.append(sorted(kernels_of(lambda: [f() for f in steps])))
    elif family == "conv_chain":
        ch = ConvChain(g)

        def conv3():
            state = ch.s0
            for t0, t1 in chunks(N_LONG, 7)[:3]:
                _, state = ch.step(state, t0, t1)
        out.append(sorted(kernels_of(conv3)))
    elif family in ("wkv6_chain", "gla_chain"):
        ch = WkvChain(g, family == "gla_chain")

        def wkv3():
            s = ch.D[-1]
            for t0, t1 in chunks(N_LONG, 7)[:3]:
                _, s = wkv_launch(g, ch.case, ch.args([a[t0:t1] for a in ch.per_tok], s))
        out.append(sorted(kernels_of(wkv3)))
    elif family == "rope_chain":
        ch = RopeChain(g)
        out.append(sorted(kernels_of(lambda: ch.run(False))))
    else:                                             # "<op>_graph": one replay of the captured chunk step
        ch = {"scan_graph": lambda: ScanChain(g), "conv_graph": lambda: ConvChain(g), "wkv6_graph": lambda: WkvChain(g, False),
              "gla_graph": lambda: WkvChain(g, True)}[family]()
        graph = ch.graph(512)[-1]
        out.append(sorted(kernels_of(graph.replay)))
    return out


def poisoned_launch(launch, n, dtype):
    """launch(out) into a poisoned buffer; checks the guards and that a relaunch into zeros gives the same bits.  Returns the result as a
    numpy array (flat)."""
    import torch
    p = Poisoned(n, dtype)
    launch(p.y)
    torch.cuda.synchronize()
    assert p.guards_ok(), "a guard band was written"
    first = p.y.clone()
    p.y.zero_()
    launch(p.y)
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int16 if dtype == torch.float16 else torch.int32),
                       p.y.view(torch.int16 if dtype == torch.float16 else torch.int32)), "relaunch into zeros differs"
    assert p.guards_ok()
    return first.cpu().numpy()


def within(what, y, r, b, report):
    q = seq.ratio(y, r, b)
    worst = float(q.max())
    report.append((worst, what))
    assert worst <= 1.0, (what, worst, int(np.argmax(q)))


def print_worst(op, rows):
    w, case = max(rows)
    print(f"{op}: worst |y - r| / bound {w:.3g} at {case}")


# ------------------------------------------------------------------ ROPE
def rope_gpu_cases():
    cases = T.rope_cases()
    # prefills: 4096 positions x 32 heads x 128, positions drawn uniformly from [0, 4096); the f32 one as llama-3.1 runs it (its freq
    # factors, base 500000)
    cases.append(R.Case(O.F32, (128, 32, 4096, 1), 128, R.ROPE_NEOX, ff=True, llama3_ff=True, freq_base=500000.0, seed=20))
    cases.append(R.Case(O.F16, (128, 32, 4096, 1), 128, R.ROPE_NORM, seed=21))
    return cases


def test_rope_elements(g):
    import torch
    ran("rope", ["rope_kernel"])
    rows, f16_flips, f16_far = [], 0, 0
    for case in rope_gpu_cases():
        x, pos, ff = case.inputs()
        xs = x.reshape(case.ne[::-1])
        p = T.params_of(case)
        r, b = seq.rope(xs, pos, p, ff)
        dt = torch.float32 if case.type == O.F32 else torch.float16
        X, P, FF = dev(xs), dev(pos), (dev(ff) if ff is not None else None)
        y = poisoned_launch(lambda out: g.op_rope(X, P, p, FF, out=out.view(X.shape)), xs.size, dt).reshape(xs.shape)
        within(str(case), y, r, b, rows)
        cpu = R.probe("CPU", case).reshape(xs.shape)
        if case.type == O.F16:
            # one f16 ulp apart, or (across zero, where the two sides can round to opposite signs) both within their bound of r
            ulp = np.spacing(np.maximum(np.abs(y), np.abs(cpu)).astype(np.float16)).astype(np.float64)
            apart = np.abs(y.astype(np.float64) - cpu.astype(np.float64))
            assert np.all((apart <= ulp) | (apart <= 2 * b)), str(case)
            f16_flips += int(np.count_nonzero(y.view(np.int16) != cpu.view(np.int16)))
            f16_far += int(np.count_nonzero(apart > ulp))
        else:
            assert np.all(np.abs(y.astype(np.float64) - cpu) <= 2 * b), str(case)
    print_worst("ROPE", rows)
    print(f"ROPE vs ggml-cpu: f16 elements that differ: {f16_flips}, of which more than one ulp apart: {f16_far}")


def test_rope_k_shift_in_place_on_a_strided_cache_view(g):
    """the K-shift: f16 ROPE in place on heads 1..6 of slots 64..447 of a [512, 8, 128] cache, by position deltas of both signs; every
    cache byte outside the view stays as it was"""
    import torch
    n_ctx, n_kv, head = 512, 8, 128
    rng = np.random.default_rng(3)
    deltas = tuple(int(v) for v in rng.integers(-300, 301, 384))
    case = R.Case(O.F16, (head, 6, 384, 1), head, R.ROPE_NEOX, inplace=True, positions=deltas, seed=30)
    x, pos, _ = case.inputs()
    xs = x.reshape(1, 384, 6, head)
    p = T.params_of(case)
    r, b = seq.rope(xs, pos, p)
    cache = torch.from_numpy(rng.uniform(-1, 1, (n_ctx, n_kv, head)).astype(np.float16)).cuda()
    view = cache[64:448, 1:7, :]
    view.copy_(dev(xs[0]))
    before = cache.clone()
    P = dev(pos)
    g.op_rope(view.unsqueeze(0), P, p, inplace=True)
    after = cache.cpu().numpy()
    ran("kshift", ["rope_kernel"])
    mask = np.zeros((n_ctx, n_kv, head), dtype=bool)
    mask[64:448, 1:7, :] = True
    assert np.array_equal(after.view(np.int16)[~mask], before.cpu().numpy().view(np.int16)[~mask]), "bytes outside the view changed"
    y = after[64:448, 1:7, :][None]
    rows = []
    within("k-shift", y, r, b, rows)
    cpu = R.probe("CPU", case).reshape(xs.shape)          # ggml-cpu's in-place form on the same values, contiguous
    ulp = np.spacing(np.maximum(np.abs(y), np.abs(cpu)).astype(np.float16)).astype(np.float64)
    apart = np.abs(y.astype(np.float64) - cpu.astype(np.float64))
    assert np.all((apart <= ulp) | (apart <= 2 * b))
    print_worst("ROPE K-shift", rows)


# ------------------------------------------------------------------ SSM_CONV
CONV = [S.ConvCase(4, 1000, 512, 4, seed=1), S.ConvCase(4, 5120, 1, 1, seed=2), S.ConvCase(4, 8192, 512, 1, seed=3), S.ConvCase(4, 8192, 1, 4, seed=4)]


def test_ssm_conv_elements(g):
    import torch
    ran("conv", ["ssm_conv_kernel"])
    rows = []
    for case in CONV:
        sx, c = seq.conv_arrays(case)
        r, b = seq.ssm_conv(sx, c)
        SX, Cw = dev(sx), dev(c)
        y = poisoned_launch(lambda out: g.op_ssm_conv(SX, Cw, out=out), r.size, torch.float32).reshape(r.shape)
        within(str(case), y, r, b, rows)
        assert np.array_equal(y.view(np.uint32), S.ssm_conv("CPU", case).view(np.uint32)), str(case)
    print_worst("SSM_CONV", rows)
    print("SSM_CONV vs ggml-cpu: bit-identical")


# ------------------------------------------------------------------ SSM_SCAN
SCAN = [S.ScanCase(16, 1000, N_LONG, 1, bc_rank=48, seed=1), S.ScanCase(16, 1536, 64, 8, bc_rank=160, seed=2),
        S.ScanCase(256, 5120, 1, 8, bc_rank=256, seed=3), S.ScanCase(256, 8192, 1, 1, bc_rank=48, seed=4),
        S.ScanCase(16, 8192, 8, 1, bc_rank=160, seed=5)]


def scan_launch(g, s0, x, dt, A, xdb, bc_rank, ds, out=None):
    """op_scan with B and C as strided views of x_db [n_s, n_t, bc_rank + 2 d_state]"""
    B = xdb[:, :, bc_rank:bc_rank + ds]
    Cc = xdb[:, :, bc_rank + ds:bc_rank + 2 * ds]
    return g.op_ssm_scan(s0, x, dt, A, B, Cc, out=out)


def scan_inputs(case):
    v = case.views()
    s0, x, dt, A = (S.read(w) for w in v[:4])
    xdb = v[4].parent
    return v, s0[0], x[0], dt[0], A[0, 0], xdb


def test_ssm_scan_elements(g):
    import torch
    ran("scan", ["ssm_scan_kernel"])
    ys, sts, ulps = [], [], []
    for case in SCAN:
        v, s0, x, dt, A, xdb = scan_inputs(case)
        ry, ey, rs, es = seq.ssm_scan(*seq.scan_arrays(case, v))
        D = [dev(a) for a in (s0, x, dt, A, xdb)]
        flat = poisoned_launch(lambda out: scan_launch(g, *D, case.bc_rank, case.d_state, out=out), ry.size + rs.size, torch.float32)
        y, st = flat[:ry.size].reshape(ry.shape), flat[ry.size:].reshape(rs.shape)
        within(str(case), y, ry, ey, ys)
        within(str(case), st, rs, es, sts)
        cy, cst = S.ssm_scan("CPU", case, v)
        assert np.all(np.abs(y - cy) <= 2 * ey) and np.all(np.abs(st - cst) <= 2 * es), str(case)
        ulps.append((max(int(S.ulps_apart(y, cy).max()), int(S.ulps_apart(st, cst).max())), str(case)))
    print_worst("SSM_SCAN y", ys)
    print_worst("SSM_SCAN states", sts)
    w = max(ulps)
    print(f"SSM_SCAN vs ggml-cpu: within the sum of both bounds everywhere, at most {w[0]} f32 ulps apart, at {w[1]}")


# ------------------------------------------------------------------ RWKV_WKV6 / GATED_LINEAR_ATTN
KEEP = T.KEEP
WKV = [W.WkvCase(40, 32, N_LONG, 1, seed=1, w_range=KEEP), W.WkvCase(64, 32, N_LONG, 1, True, 1.0, seed=2, w_range=KEEP),
       W.WkvCase(80, 40, 16, 3, seed=3), W.WkvCase(128, 40, 1, 8, True, 64 ** -0.5, seed=4), W.WkvCase(200, 32, 4, 3, True, 1.0, seed=5),
       W.WkvCase(256, 64, 1, 3, seed=6), W.WkvCase(256, 32, 2, 1, True, 64 ** -0.5, seed=7), W.WkvCase(40, 64, 1, 8, True, 1.0, seed=8),
       W.WkvCase(200, 40, 1, 1, seed=9)]


def wkv_launch(g, case, D, out=None):
    if case.gla:
        return g.op_gated_linear_attn(*D, case.scale, out=out)
    return g.op_rwkv_wkv6(*D, out=out)


def test_wkv_elements(g):
    import torch
    ys, sts, same, tails = [], [], [], []
    ran("wkv", ["wkv_kernel"])
    for case in WKV:
        srcs = case.sources()
        ry, ey, rs, es = seq.wkv(*seq.wkv_args(case, srcs))
        D = [dev(a) for a in srcs]
        flat = poisoned_launch(lambda out: wkv_launch(g, case, D, out=out), ry.size + rs.size, torch.float32)
        y, st = flat[:ry.size].reshape(ry.shape), flat[ry.size:].reshape(rs.shape)
        within(str(case), y, ry, ey, ys)
        within(str(case), st, rs, es, sts)
        cy, cst = W.wkv("CPU", case, srcs)
        if case.S % 16 == 0:
            assert np.array_equal(y.view(np.uint32), cy.view(np.uint32)) and np.array_equal(st.view(np.uint32), cst.view(np.uint32)), str(case)
            same.append(str(case))
        else:
            assert np.all(np.abs(y - cy) <= 2 * ey) and np.all(np.abs(st - cst) <= 2 * es), str(case)
            tails.append((float(max(seq.ratio(y, cy, 2 * ey).max(), seq.ratio(st, cst, 2 * es).max())), str(case)))
    print_worst("WKV y", ys)
    print_worst("WKV states", sts)
    w = max(tails)
    print(f"WKV vs ggml-cpu: bit-identical in {len(same)} cases (S % 16 == 0); the others within the sum of both bounds, "
          f"worst |y - cpu| / (2 bound) {w[0]:.3g} at {w[1]}")


# ------------------------------------------------------------------ chunk invariance and dependent launches
def chunks(n, c):
    return [(t, min(t + c, n)) for t in range(0, n, c)]


def _bits(t):
    import torch
    return t.contiguous().view(torch.int32)


def run_chain(steps, sync):
    """run the chunk steps in order (each returns its outputs); sync: torch.cuda.synchronize() after each launch"""
    import torch
    outs = []
    for step in steps:
        outs.append(step())
        if sync:
            torch.cuda.synchronize()
    torch.cuda.synchronize()
    return outs


class ScanChain:
    def __init__(self, g):
        self.g = g
        self.case = S.ScanCase(16, 1000, N_LONG, 1, bc_rank=48, seed=11)
        _, s0, x, dt, A, xdb = scan_inputs(self.case)
        self.s0, self.x, self.dt, self.A, self.xdb = (dev(a) for a in (s0, x, dt, A, xdb))

    def whole(self):
        return scan_launch(self.g, self.s0, self.x, self.dt, self.A, self.xdb, 48, 16)

    def steps(self, c):
        """the chunk steps of a c-token chunking; each launches one ssm_scan_kernel and nothing else (x and dt are passed as views that
        are already packed for one sequence, B and C as strided views of x_db), so the chain is scan after scan"""
        state = [self.s0]
        ys = []

        def step(t0, t1):
            def f():
                y, st = scan_launch(self.g, state[0], self.x[0, t0:t1].unsqueeze(0), self.dt[0, t0:t1].unsqueeze(0), self.A,
                                    self.xdb[:, t0:t1], 48, 16)
                state[0] = st
                ys.append(y)
                return y
            return f
        return [step(*b) for b in chunks(N_LONG, c)], ys, state


    def graph(self, c):
        """one c-token chunk step captured as a CUDA graph over static buffers: (load(t0, t1), replay() -> y, the state buffer it reads
        and writes, restart(), the graph)"""
        import torch
        g = self.g
        sx, sdt, sxdb = packed(self.x[:, :c]), packed(self.dt[:, :c]), packed(self.xdb[:, :c])
        s_in = self.s0.clone()
        scan_launch(g, s_in, sx, sdt, self.A, sxdb, 48, 16)                     # set-up outside the capture
        torch.cuda.synchronize()
        graph, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        with torch.cuda.graph(graph, stream=stream):
            gy, gst = scan_launch(g, s_in, sx, sdt, self.A, sxdb, 48, 16)

        def load(t0, t1):
            sx.copy_(self.x[:, t0:t1]); sdt.copy_(self.dt[:, t0:t1]); sxdb.copy_(self.xdb[:, t0:t1])

        def replay():
            graph.replay()
            y = gy.clone()
            s_in.copy_(gst)
            return y
        return load, replay, s_in, lambda: s_in.copy_(self.s0), graph


def test_scan_chunked_prompt_is_bit_identical(g):
    import torch
    ran("scan_chain", ["ssm_scan_kernel"], only=True)
    ch = ScanChain(g)
    y, st = ch.whole()
    torch.cuda.synchronize()
    for c in CHUNKS:                                     # each chain back to back: scan after scan, nothing in between
        steps, ys, state = ch.steps(c)
        run_chain(steps, sync=False)
        assert torch.equal(_bits(torch.cat(ys, 1)), _bits(y)), c
        assert torch.equal(_bits(state[0]), _bits(st)), c
    # dependent launches: the chunk-7 chain back to back equals the same chain synchronised after every launch
    steps, ys_a, st_a = ch.steps(7)
    run_chain(steps, sync=True)
    steps, ys_b, st_b = ch.steps(7)
    run_chain(steps, sync=False)
    assert torch.equal(_bits(torch.cat(ys_a, 1)), _bits(torch.cat(ys_b, 1))) and torch.equal(_bits(st_a[0]), _bits(st_b[0]))


def test_scan_graph_replay_over_chunks(g):
    import torch
    ran("scan_graph", ["ssm_scan_kernel"], only=True)
    ch = ScanChain(g)
    y, st = ch.whole()
    load, replay, s_in, restart, _ = ch.graph(512)
    restart()
    outs = []
    for t0, t1 in chunks(N_LONG, 512):
        load(t0, t1)
        outs.append(replay())
    torch.cuda.synchronize()
    assert torch.equal(_bits(torch.cat(outs, 1)), _bits(y)) and torch.equal(_bits(s_in), _bits(st))


class ConvChain:
    """the Mamba layer's conv: conv_x = CONCAT(the previous conv_x's last d_conv − 1 columns, x transposed), then SSM_CONV"""

    def __init__(self, g):
        self.g = g
        rng = np.random.default_rng(12)
        self.d_conv, self.d_inner, self.n_s = 4, 1000, 4
        self.x = dev(rng.standard_normal((self.n_s, N_LONG, self.d_inner)).astype(np.float32))          # [n_s, n_t, d_inner]
        self.c = dev((rng.standard_normal((self.d_inner, self.d_conv)) / 2).astype(np.float32))
        self.s0 = dev(rng.standard_normal((self.n_s, self.d_inner, self.d_conv - 1)).astype(np.float32))

    def step(self, state, t0, t1):
        cx = self.g.op_concat(state, self.x[:, t0:t1].transpose(1, 2), 0)
        return self.g.op_ssm_conv(cx, self.c), cx[:, :, -(self.d_conv - 1):]

    def run(self, c, sync):
        import torch
        state, ys = self.s0, []
        for t0, t1 in chunks(N_LONG, c):
            y, state = self.step(state, t0, t1)
            ys.append(y)
            if sync:
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        return torch.cat(ys, 1), state.contiguous()

    def graph(self, c):
        """one c-token chunk step (CONCAT, SSM_CONV) captured as a CUDA graph: as ScanChain.graph"""
        import torch
        g = self.g
        s_in, sxc = self.s0.clone(), torch.empty((self.n_s, c, self.d_inner), dtype=torch.float32, device="cuda")
        cx = torch.empty((self.n_s, self.d_inner, self.d_conv - 1 + c), dtype=torch.float32, device="cuda")
        gy = torch.empty((self.n_s, c, self.d_inner), dtype=torch.float32, device="cuda")

        def step():
            g.op_concat(s_in, sxc.transpose(1, 2), 0, out=cx)
            g.op_ssm_conv(cx, self.c, out=gy)
        step()
        torch.cuda.synchronize()
        graph, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        with torch.cuda.graph(graph, stream=stream):
            step()

        def replay():
            graph.replay()
            y = gy.clone()
            s_in.copy_(cx[:, :, -(self.d_conv - 1):])
            return y
        return (lambda t0, t1: sxc.copy_(self.x[:, t0:t1])), replay, s_in, lambda: s_in.copy_(self.s0), graph


def test_conv_chunked_prompt_is_bit_identical(g):
    import torch
    ran("conv_chain", ["concat_kernel", "ssm_conv_kernel"], only=True)
    ran("conv_graph", ["concat_kernel", "ssm_conv_kernel"], only=True)
    ch = ConvChain(g)
    y, st = ch.run(N_LONG, sync=True)
    sx = torch.cat([ch.s0, ch.x.transpose(1, 2)], 2).cpu().numpy()
    r, b = seq.ssm_conv(sx, ch.c.cpu().numpy())
    within("conv chain", y.cpu().numpy(), r, b, [])
    for c in CHUNKS:
        yc, stc = ch.run(c, sync=False)
        assert torch.equal(_bits(yc), _bits(y)) and torch.equal(_bits(stc), _bits(st)), c
    ya, sa = ch.run(7, sync=True)
    yb, sb = ch.run(7, sync=False)
    assert torch.equal(_bits(ya), _bits(yb)) and torch.equal(_bits(sa), _bits(sb))
    # one chunk step captured as a CUDA graph, replayed over the 512-token chunks
    load, replay, s_in, restart, _ = ch.graph(512)
    restart()
    outs = []
    for t0, t1 in chunks(N_LONG, 512):
        load(t0, t1)
        outs.append(replay())
    torch.cuda.synchronize()
    assert torch.equal(_bits(torch.cat(outs, 1)), _bits(y)) and torch.equal(_bits(s_in), _bits(st))


class WkvChain:
    """a 2048-token WKV6 / GLA prompt (S 64, H 32, decays up to 1 − 3e-4) as one call and as chunks, each chunk's final state the next's s0"""

    def __init__(self, g, gla: bool):
        self.g = g
        self.case = W.WkvCase(64, 32, N_LONG, 1, gla, 64 ** -0.5 if gla else 1.0, seed=13, w_range=KEEP)
        self.D = [dev(a) for a in self.case.sources()]
        self.per_tok = [a for a in self.D[:-1] if a.shape[0] == N_LONG]
        self.fixed = [a for a in self.D[:-1] if a.shape[0] != N_LONG]          # tf (WKV6)

    def args(self, toks, s):
        return (toks[:3] + self.fixed + toks[3:] + [s]) if not self.case.gla else (toks + [s])

    def whole(self):
        return wkv_launch(self.g, self.case, self.D)

    def chain(self, c, sync):
        """the c-token chunking, launch after launch (only wkv_kernel: the token slices are views)"""
        import torch
        s, ys = self.D[-1], []
        for t0, t1 in chunks(N_LONG, c):
            yy, s = wkv_launch(self.g, self.case, self.args([a[t0:t1] for a in self.per_tok], s))
            ys.append(yy)
            if sync:
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        return torch.cat(ys, 0), s

    def graph(self, c):
        import torch
        stat = [packed(a[:c]) for a in self.per_tok]
        s_in = self.D[-1].clone()
        sargs = self.args(stat, s_in)
        wkv_launch(self.g, self.case, sargs)
        torch.cuda.synchronize()
        graph, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        with torch.cuda.graph(graph, stream=stream):
            gy, gs = wkv_launch(self.g, self.case, sargs)

        def load(t0, t1):
            for a, b in zip(stat, self.per_tok):
                a.copy_(b[t0:t1])

        def replay():
            graph.replay()
            y = gy.clone()
            s_in.copy_(gs)
            return y
        return load, replay, s_in, lambda: s_in.copy_(self.D[-1]), graph


@pytest.mark.parametrize("gla", [False, True], ids=["wkv6", "gla"])
def test_wkv_chunked_prompt_dependent_launches_and_graph_replay(g, gla):
    import torch
    name = "gla" if gla else "wkv6"
    ran(f"{name}_chain", ["wkv_kernel"], only=True)
    ran(f"{name}_graph", ["wkv_kernel"], only=True)
    ch = WkvChain(g, gla)
    y, st = ch.whole()
    torch.cuda.synchronize()
    for c in CHUNKS:
        yc, sc = ch.chain(c, sync=False)
        assert torch.equal(_bits(yc), _bits(y)) and torch.equal(_bits(sc), _bits(st)), c
    ya, sa = ch.chain(7, sync=True)
    yb, sb = ch.chain(7, sync=False)
    assert torch.equal(_bits(ya), _bits(yb)) and torch.equal(_bits(sa), _bits(sb))
    load, replay, s_in, restart, _ = ch.graph(512)
    restart()
    outs = []
    for t0, t1 in chunks(N_LONG, 512):
        load(t0, t1)
        outs.append(replay())
    torch.cuda.synchronize()
    assert torch.equal(_bits(torch.cat(outs, 0)), _bits(y)) and torch.equal(_bits(s_in), _bits(st))


class RopeChain:
    """three ROPEs back to back, each rotating the previous one's output"""

    def __init__(self, g):
        self.g = g
        rng = np.random.default_rng(14)
        self.x = dev(rng.uniform(-1, 1, (2, 512, 32, 128)).astype(np.float32))
        self.pos = [dev(rng.integers(-(1 << 20), 1 << 20, 512).astype(np.int32)) for _ in range(3)]
        self.p = g.rope_params(128, g.ROPE_NEOX, n_ctx_orig=8192, freq_scale=0.125, ext_factor=1.0, attn_factor=1.1)

    def run(self, sync):
        import torch
        y = self.x
        for q in self.pos:
            y = self.g.op_rope(y, q, self.p)
            if sync:
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        return y


def test_rope_dependent_chain_matches_synchronised(g):
    """the ROPE chain back to back against the same launches synchronised"""
    import torch
    ran("rope_chain", ["rope_kernel"], only=True)
    ch = RopeChain(g)
    assert torch.equal(_bits(ch.run(True)), _bits(ch.run(False)))
