"""GPU: every mat-mul route checked on every output element against the f64 reference of oracle/mm.py, through poisoned buffers.

Routes: every entry of tests/test_mul_mat_routes.py::AGREE_MM, plus mul_mat_f16, mul_mat_f16_f16, the fused epilogue and MUL_MAT_ID
(the expert-grouped MUL_MAT_ID runs in tests/gpu_mmid_grouped_check.py, in its own process).  Each route gets a grid over M (1 and the
16- and 256-row tile edges, ragged), K (one unit, long, K % 256 != 0 where the route takes it), N (the route's range), the flags
SRC0_STATIC and SRC0 | SRC1_STATIC, src1 contiguous or with padded rows (16 bytes; 4 bytes with a base that is only 4-byte aligned,
wherever the planner accepts it), and activation rows that are zero or scaled by 2^-16, 2^-20 and 2^-30.  Every case runs with the
flags that force its route's kernel, and which kernels it launched is read back with torch.profiler: a case the planner refuses or
hands to a sibling kernel does not count for the route, and each route reports those cases.

Every launch writes into the middle of a larger buffer: guard bands either side hold a NaN sentinel bit pattern, dst holds NaN, and the
workspace is exactly the queried size, filled with 0xFF and followed by a guard band.  After the launch every element must lie within
the bound (oracle/mm.py), every 256 x 64 block and every column within the NMSE gates, the guard bands, W and X unchanged.  A second
launch into zeros (dst and workspace) must give the same bits.

Dependent chains: mat-muls (and op_norm) enqueued on one stream with one shared workspace and no host synchronisation, each output
the next launch's src1, every intermediate NaN-filled on the stream first; every output must be bitwise identical to the same launches
run with a synchronisation between them, and each launch of the synchronised run is checked to run on its route's kernel.

Large shapes (vocabulary-sized M, dst over 2^31 bytes, an expert stack over 2^31 bytes with tokens on experts past that offset) run
when the GPU has the free memory, and skip saying how much there was otherwise.  The whole file takes a few minutes on one H100."""
import ctypes as C

import numpy as np
import pytest

from oracle import mm
from oracle import oracle as O
import test_mul_mat_routes as R

pytestmark = pytest.mark.gpu

GUARD = 4096                          # guard band, in elements (floats) or bytes (workspace)
SENTINEL = 0x7FC0DEAD                 # a NaN no kernel writes
WS_SENTINEL = 0xA5
# gates, about 10x the worst measured on an H100 80GB HBM3 at 700 W (DESIGN.md §5): per-element |y - r| / bound (worst 0.0111 on the
# integer-dot routes; 0.206 on the fp16 routes, where the gate is the bound itself), NMSE per 256 x 64 block and per column (worst
# 2.7e-14 integer-dot, 4.7e-7 fp16)
RATIO_GATE = {"int": 0.1, "f16": 1.0}
NMSE_GATE = {"int": 3e-13, "f16": 5e-6}
FAMILY = {"generic": 1, "first-generation TMA": 2, "superblock": 2, "mma": 2, "wgmma": 4, "dense": 4}
SPECIAL = (0.0, 2.0 ** -16, 2.0 ** -20, 2.0 ** -30)


def route_family(name: str) -> str:
    return next(k for k in FAMILY if name.startswith(k))


@pytest.fixture(scope="module")
def env():
    import torch
    import ggml_b200 as g
    assert torch.cuda.is_available(), "these tests need an H100"
    L = R.load(g.KERNELS_SO)
    L.ggml_b200_mul_mat_f16_f16_workspace_size.restype = C.c_size_t
    L.ggml_b200_mul_mat_f16_f16_workspace_size.argtypes = [C.c_int64] * 3
    L.ggml_b200_mul_mat_f16_f16.argtypes = L.ggml_b200_mul_mat_f16.argtypes
    return g, L, O.Oracle()


def stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------------------------------------------------------- poisoned buffers
class Poisoned:
    """n f32 elements in the middle of a buffer with NaN-sentinel guard bands; .fill(v) refills the middle, .guards_ok() checks the bands"""

    def __init__(self, n: int):
        import torch
        self.buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int32, device="cuda")
        self.n = n
        self.y = self.buf[GUARD:GUARD + n].view(torch.float32)

    def fill(self, v: float):
        self.y.fill_(v)
        return self

    def guards_ok(self) -> bool:
        return bool((self.buf[:GUARD] == SENTINEL).all()) and bool((self.buf[GUARD + self.n:] == SENTINEL).all())


class Scratch:
    """a workspace of exactly `n` bytes followed by a guard band"""

    def __init__(self, n: int):
        import torch
        self.buf = torch.full((n + GUARD,), WS_SENTINEL, dtype=torch.uint8, device="cuda")
        self.n = n
        self.ws = self.buf[:n]

    def fill(self, v: int):
        self.ws.fill_(v)
        return self

    def guards_ok(self) -> bool:
        return bool((self.buf[self.n:] == WS_SENTINEL).all())


def src1_buffer(X: np.ndarray, layout: str):
    """X [N, K] on the device as `layout`: (keep-alive tensor, data pointer, row stride in bytes)"""
    import torch
    N, K = X.shape
    if layout == "contig":
        t = torch.from_numpy(np.ascontiguousarray(X)).cuda()
        return t, t.data_ptr(), K * 4
    pad = {"pad16": 4, "pad4": 1}[layout]
    base = 1 if layout == "pad4" else 0                  # one float in: the base is 4-byte aligned only
    t = torch.full((base + N * (K + pad),), float("nan"), dtype=torch.float32, device="cuda")
    t[base:].view(N, K + pad)[:, :K] = torch.from_numpy(np.ascontiguousarray(X)).cuda()
    return t, t.data_ptr() + base * 4, (K + pad) * 4


def activations(rng, N: int, K: int, special: int | None = None) -> np.ndarray:
    """uniform(-1, 1) rows; with N >= 5 the last four rows are zero and scaled by 2^-16, 2^-20 and 2^-30; with fewer rows, `special` i
    makes the last row SPECIAL[i % 4] times its values"""
    X = rng.uniform(-1, 1, (N, K)).astype(np.float32)
    if N >= 5:
        for i, s in enumerate(SPECIAL):
            X[N - 1 - i] *= np.float32(s)
    elif special is not None:
        X[N - 1] *= np.float32(SPECIAL[special % 4])
    return X


def check_values(what, y, r, bound, kind, report):
    q = mm.ratio(y, r, bound)
    worst = float(q.max())
    blk, col = mm.nmse_blocks(y, r)
    report.append((what, kind, worst, blk, col))
    assert worst <= RATIO_GATE[kind], f"{what}: |y - r| / bound = {worst:.3g} at (n, m) = {np.unravel_index(int(q.argmax()), tuple(q.shape))}"
    assert blk <= NMSE_GATE[kind] and col <= NMSE_GATE[kind], f"{what}: block NMSE {blk:.3g}, column NMSE {col:.3g} > {NMSE_GATE[kind]}"


def kernel_names(fn) -> list[str]:
    """the names of the CUDA kernels fn launches (torch.profiler)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def launch_twice(what, launch, sizes, ws_size: int, inputs, profile: bool = False):
    """launch(outs, ws) with outs one f32 tensor per entry of `sizes`, all NaN inside NaN-sentinel guard bands, and ws a uint8 tensor of
    exactly ws_size bytes (0xFF, then a guard band); then again into zeros.  Checks the guards, the inputs and the bits of the two
    launches; returns (clones of the first launch's outputs, the kernel names of both launches when profile, else None)."""
    import torch
    outs, ws = [Poisoned(n).fill(float("nan")) for n in sizes], Scratch(ws_size).fill(0xFF)
    before = [t.clone() for t in inputs]
    names = None
    if profile:
        names = kernel_names(lambda: launch([o.y for o in outs], ws.ws))
    else:
        launch([o.y for o in outs], ws.ws)
    torch.cuda.synchronize()
    assert all(o.guards_ok() for o in outs), f"{what}: a write outside dst"
    assert ws.guards_ok(), f"{what}: a write past the workspace it asked for"
    assert all(torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(before, inputs)), f"{what}: an input changed"
    first = [o.y.clone() for o in outs]
    for o in outs:
        o.fill(0.0)
    ws.fill(0x00)
    if profile:                                          # the profiler has been seen to drop a kernel record: both launches' names count
        names += kernel_names(lambda: launch([o.y for o in outs], ws.ws))
    else:
        launch([o.y for o in outs], ws.ws)
    torch.cuda.synchronize()
    for y1, o in zip(first, outs):
        assert torch.equal(y1.view(torch.int32), o.y.view(torch.int32)), f"{what}: not the same bits after zero-filled dst and workspace"
    return first, names


def ptr(t):
    """device address of a tensor for the C ABI, None for an empty one"""
    return t.data_ptr() if t.numel() else None


# ---------------------------------------------------------------------------------------------------------------- the route grid
def force_flags(g, fam: str) -> int:
    """the flags that select the route's kernel (the planner falls back to a sibling where that kernel cannot take the shape)"""
    return {"generic": g.MM_GENERIC, "first-generation TMA": g.MM_GEMV | g.MM_GEMV_V1, "superblock": g.MM_GEMV | g.MM_GEMV_DP4A,
            "mma": g.MM_GEMV | g.MM_GEMV_MMA, "wgmma": g.MM_GEMM, "dense": g.MM_GEMM}[fam]


def ran_on(names: list[str]) -> str:
    """the route a launch took, from its kernel names"""
    has = lambda k: any(k in n for n in names)                               # noqa: E731
    if has("mmq_tc2_kernel"):
        return "dense" if has("dequantize") else "wgmma"
    for k, fam in (("mmvq_mma_kernel", "mma"), ("mmvq_sb_kernel", "superblock"), ("mmvq_tma_kernel", "first-generation TMA"),
                   ("mmvq_generic_kernel", "generic")):
        if has(k):
            return fam
    return "none of the mat-mul kernels: " + ", ".join(sorted(set(names)))


def route_cases(t, M0, N0, K0, flags0, fam):
    """(M, N, K) per case: M edges and ragged at the route's N and K; K variants; N over the route's range"""
    qk = R.qk(t)
    if fam in ("wgmma", "dense"):
        Ms = [1, 255, 256, 257, 1000]
        Ns = [n for n in (9, 15, 63, 64, 65, 127, 128, 129, 1024, 4096) if n >= (5 if flags0 & 4 else 9)] + ([5, 8] if flags0 & 4 else [])
        Ks = [256, 16384 if fam == "wgmma" and O.Oracle().row_size(t, 16384) % 16 == 0 else 14336]
    else:
        Ms = [1, 15, 16, 17, 1000, 4099]
        Ns = {"generic": [1, 2, 5, 9, 33], "first-generation TMA": [1], "superblock": [N0] if N0 > 1 else [1],
              "mma": [1, 2, 3, 5, 8]}[fam]
        if fam == "superblock" and N0 > 1:
            Ns = [2, 3, 4, 6, 8]
        Ks = [256, 14336, 16384] + ([4128] if qk == 32 else []) + ([qk] if fam == "generic" and qk == 32 else [])
        if fam == "mma":                                 # its planner's limits: K >= 2048 and M >= one 16-row tile (M = 15: the edge below)
            Ms, Ks = [15, 16, 17, 1000, 4099], [2048, 14336, 16384]
    cases = [(M, N0, K0) for M in Ms] + [(M0, N0, K) for K in Ks] + [(M0 if N < 1024 else 1024, N, K0) for N in Ns if N != N0]
    return cases


@pytest.mark.parametrize("entry", R.AGREE_MM, ids=[f"{O.TYPE_NAMES[e[0]]}-{e[5].replace(' ', '_').replace(',', '')}" for e in R.AGREE_MM])
def test_route_elements(entry, env, report):
    """Each case runs with the route's forcing flags, and its kernels are read back with torch.profiler.  A case the planner refuses, or
    one it hands to a sibling kernel, is still checked on its values but does not count for the route, and it is reported."""
    import torch
    g, L, orc = env
    t, M0, N0, K0, flags0, name = entry
    fam = route_family(name)
    kind = "f16" if fam in ("wgmma", "dense") else "int"
    rng = np.random.default_rng(t * 1000 + M0 + N0)
    ran, missed = 0, []
    weights = {}
    for i, (M, N, K) in enumerate(route_cases(t, M0, N0, K0, flags0, fam)):
        flags = flags0 | force_flags(g, fam) | (g.MM_SRC0_STATIC if i % 2 == 0 else g.MM_SRC0_STATIC | g.MM_SRC1_STATIC)
        layout = ("contig", "pad16") [i % 2] if fam == "mma" else ("contig", "pad16", "pad4")[i % 3]     # mma: 16-byte aligned src1 only
        if (M, K) not in weights:
            weights.clear()
            W = O.random_blocks(t, M * K // R.qk(t), rng)
            weights[(M, K)] = (torch.from_numpy(W).cuda(), mm.Reference(orc, t, W, M, K, device="cuda"))
        Wd, ref = weights[(M, K)]
        X = activations(rng, N, K, special=i // 3 if i % 3 == 0 else None)
        for lay in (layout, "contig"):
            xt, xp, nb11 = src1_buffer(X, lay)
            a = R.mm_args(L, t, M, N, K, flags, xp)
            a.nb11, a.nb12, a.nb13 = nb11, nb11 * N, nb11 * N
            a.src0 = Wd.data_ptr()
            if int(L.ggml_b200_mul_mat_plan(C.byref(a))) == FAMILY[fam]:
                break
            missed.append((M, N, K, flags, lay, "refused by the planner"))
        else:
            continue
        ws_size = int(L.ggml_b200_mul_mat_workspace_size(C.byref(a)))

        def launch(outs, ws, a=a):
            a.dst, a.workspace, a.workspace_size = outs[0].data_ptr(), ptr(ws), ws.numel()
            g.check(L.ggml_b200_mul_mat(C.byref(a), stream()), "ggml_b200_mul_mat")
        what = f"{name} {O.TYPE_NAMES[t]} M={M} N={N} K={K} flags={flags} src1={lay}"
        (y,), names = launch_twice(what, launch, [N * M], ws_size, [Wd, xt], profile=True)
        check_values(what, y.view(N, M), *ref(X, kind), kind, report)
        took = ran_on(names)
        if took == fam:
            ran += 1
        else:
            missed.append((M, N, K, flags, lay, f"ran on {took}"))
    print(f"\n{name} {O.TYPE_NAMES[t]}: {ran} cases on the route's kernel; not on it: {missed or 'none'}")
    assert ran >= 8, f"{name}: only {ran} cases ran on the route's kernel; the others: {missed}"


def test_f16_routes_elements(env, report):
    """mul_mat_f16 (fp16 weights x f32 activations) and mul_mat_f16_f16 (both fp16) on the wgmma GEMM"""
    import torch
    g, L, orc = env
    rng = np.random.default_rng(16)
    for M, N, K in [(1, 9, 256), (255, 64, 4096), (257, 65, 256), (1000, 129, 4096), (4096, 1024, 1024), (300, 4096, 512)]:
        Wh = torch.from_numpy(rng.uniform(-1, 1, (M, K)).astype(np.float16)).cuda()
        X = activations(rng, N, K)
        ref = mm.Reference(orc, O.F16, Wh.cpu().numpy(), M, K, device="cuda")
        xt, xp, nb11 = src1_buffer(X, "pad16")
        ws = int(L.ggml_b200_mul_mat_f16_workspace_size(M, N, K))
        assert ws > 0

        def launch(outs, wsb):
            g.check(L.ggml_b200_mul_mat_f16(Wh.data_ptr(), K * 2, xp, nb11, outs[0].data_ptr(), M, N, K, ptr(wsb), wsb.numel(), g.MM_SRC0_STATIC,
                                            stream()), "mul_mat_f16")
        (y,), names = launch_twice(f"mul_mat_f16 M={M} N={N} K={K}", launch, [N * M], ws, [Wh, xt], profile=True)
        assert ran_on(names) == "wgmma", names
        check_values(f"mul_mat_f16 M={M} N={N} K={K}", y.view(N, M), *ref(X, "f16"), "f16", report)
        # f16 x f16: x is already fp16, so the reference takes those values exactly (no prescale, no rounding)
        Xh = torch.from_numpy(X.astype(np.float16)).cuda()
        Xh[N - 4:] = 0                                   # the scaled rows underflow fp16 differently: zero them
        ws = int(L.ggml_b200_mul_mat_f16_f16_workspace_size(M, N, K))
        assert ws > 0

        def launch16(outs, wsb):
            g.check(L.ggml_b200_mul_mat_f16_f16(Wh.data_ptr(), K * 2, Xh.data_ptr(), K * 2, outs[0].data_ptr(), M, N, K, ptr(wsb), wsb.numel(), 0,
                                                stream()), "mul_mat_f16_f16")
        (y,), names = launch_twice(f"mul_mat_f16_f16 M={M} N={N} K={K}", launch16, [N * M], ws, [Wh, Xh], profile=True)
        assert ran_on(names) == "wgmma", names
        check_values(f"mul_mat_f16_f16 M={M} N={N} K={K}", y.view(N, M), *ref(Xh.float().cpu().numpy(), "f16"), "f16", report)


@pytest.mark.parametrize("t", [O.Q4_0, O.Q4_K, O.Q6_K, O.Q8_0], ids=["q4_0", "q4_K", "q6_K", "q8_0"])
def test_fused_epilogue_elements(t, env, report):
    """the fused MUL_MAT + bias + GELU epilogue, into three poisoned outputs and a poisoned workspace: y on every element within the
    bound, y + bias and GELU exactly the separate ops, the same bits when relaunched into zeros; the activation row is normal or
    zero or scaled by 2^-16, 2^-20 or 2^-30"""
    import torch
    g, L, orc = env
    rng = np.random.default_rng(t)
    shapes = [(16, 256), (17, 4096), (3072, 1024), (4099, 4096)]
    for i, (M, K) in enumerate(shapes + [(1000, 4096)] * 4):
        W = O.random_blocks(t, M * K // R.qk(t), rng)
        X = activations(rng, 1, K, special=i - len(shapes) if i >= len(shapes) else None)
        bias = torch.from_numpy(rng.uniform(-0.5, 0.5, M).astype(np.float32)).cuda()
        Wd, Xd = torch.from_numpy(W).cuda(), torch.from_numpy(X).cuda()
        a = R.mm_args(L, t, M, 1, K, 0, Xd.data_ptr())
        ws_size = int(L.ggml_b200_mul_mat_workspace_size(C.byref(a)))

        def launch(outs, ws):
            g.mul_mat_fused(t, Wd, Xd, M, K, bias, gelu=True, out=outs, workspace=ws)
        what = f"fused {O.TYPE_NAMES[t]} M={M} K={K}"
        (y, y2, y3), _ = launch_twice(what, launch, [M, M, M], ws_size, [Wd, Xd, bias])
        check_values(what, y.view(1, M), *mm.Reference(orc, t, W, M, K, device="cuda")(X, "int"), "int", report)
        assert torch.equal(y2, y + bias) and torch.equal(y3, g.op_unary(0, y + bias)), what


# ---------------------------------------------------------------------------------------------------------------- MUL_MAT_ID
def test_mul_mat_id_elements(env, report):
    """per-pair MUL_MAT_ID: 256 experts, 8 used, nb1cols 1 and 8, ids a strided view of wider rows, an expert with no tokens (200) and
    one with more than a GEMM tile of them (3), and ids -1 and n_expert whose rows must be exactly zero"""
    import torch
    g, L, orc = env
    rng = np.random.default_rng(256)
    t, ne, nu, M, K, ntok = O.Q4_K, 256, 8, 272, 2048, 160
    W = O.random_blocks(t, ne * M * K // 256, rng)
    Wd = torch.from_numpy(W).cuda()
    ref = mm.Reference(orc, t, W, ne * M, K, device="cuda")
    others = np.delete(np.arange(ne), [3, 200])
    wide = np.stack([rng.permutation(others)[:nu + 3] for _ in range(ntok)]).astype(np.int32)
    wide[:140, 0] = 3                                     # expert 3: 140 tokens (> 128, the widest tile)
    wide[5, 2], wide[9, 7], wide[100, 1] = -1, ne, -1
    used = wide[:, :nu]
    assert not (used == 200).any() and (used == 3).sum() == 140
    ids = torch.from_numpy(wide).cuda()[:, :nu]             # a strided view: row stride nu + 3
    for nb1 in (1, nu):
        X = activations(rng, ntok * nb1, K)
        xt = torch.from_numpy(X).cuda()
        a = R.mmid_args(L, t, M, K, ne, nu, nb1, ntok)
        ws_size = int(L.ggml_b200_mul_mat_id_workspace_size(C.byref(a)))

        def launch(outs, ws):
            g.mul_mat_id(t, Wd, xt, ids, M, K, ne, nu, nb1, ntok, out=outs[0], workspace=ws)
        what = f"mul_mat_id q4_K {ne}x{nu} nb1cols={nb1}"
        (y,), _ = launch_twice(what, launch, [ntok * nu * M], ws_size, [Wd, xt, ids])
        y = y.view(ntok, nu, M)
        bad = (used < 0) | (used >= ne)
        assert bad.sum() == 3 and bool((y[torch.from_numpy(bad).cuda()] == 0).all()), f"{what}: invalid-id rows are not zero"
        Xr = X.reshape(ntok, nb1, K)
        worst = 0.0
        for tok in range(ntok):
            for e in range(nu):
                x = int(wide[tok, e])
                if 0 <= x < ne:
                    r, bound = ref(Xr[tok, e % nb1][None], "int", rows=np.arange(x * M, (x + 1) * M))
                    worst = max(worst, float(mm.ratio(y[tok, e][None], r, bound).max()))
        report.append((what, "int", worst, 0.0, 0.0))
        assert worst <= RATIO_GATE["int"], f"{what}: |y - r| / bound = {worst:.3g}"


# ---------------------------------------------------------------------------------------------------------------- dependent chains
class Step:
    """one launch of a chain: fn(x_in, out, workspace); `route` is the kernel family it must run on (None: op_norm)"""

    def __init__(self, name, shape_out, route, fn, splitk=None):
        self.name, self.shape_out, self.route, self.fn, self.splitk = name, shape_out, route, fn, splitk

    def __call__(self, x, out, ws):
        self.fn(x, out, ws)


def run_chain(steps, x0, ws, sync: bool):
    """every intermediate is NaN-filled on the stream, then the steps are enqueued; sync: a synchronisation after each step, whose kernels
    are read back and checked against the step's route"""
    import torch
    outs = [torch.full(s.shape_out, float("nan"), dtype=torch.float32, device="cuda") for s in steps]
    x = x0
    for s, o in zip(steps, outs):
        if sync:
            names = kernel_names(lambda: s(x, o, ws))
            if not names:                                # a dropped profiler record: the step is idempotent, so run it once more
                names = kernel_names(lambda: s(x, o, ws))
            took = ran_on(names)
            assert (took == s.route) if s.route else any("norm" in n for n in names), f"{s.name} ran on {took}: {sorted(set(names))}"
        else:
            s(x, o, ws)
        x = o
    torch.cuda.synchronize()
    return outs


def mm_step(g, t, W, M, K, N, flags, route, splitk=None):
    def fn(x, out, ws):
        g.mul_mat(t, W, x, M, N, K, flags=flags, out=out.view(1, 1, N, M), workspace=ws)
    st = Step(f"{route} {O.TYPE_NAMES[t]} {K}->{M} n={N}", (N, M), route, fn, splitk)
    st.mm = (t, M, N, K)
    return st


def f16_step(L, g, Wh, M, K, N):
    def fn(x, out, ws):
        g.check(L.ggml_b200_mul_mat_f16(Wh.data_ptr(), K * 2, x.data_ptr(), K * 4, out.data_ptr(), M, N, K, ws.data_ptr(), ws.numel(),
                                        g.MM_SRC0_STATIC, stream()), "mul_mat_f16")
    return Step(f"mul_mat_f16 {K}->{M} n={N}", (N, M), "wgmma", fn)


def norm_step(g, shape):
    def fn(x, out, ws):                                  # RMS_NORM straight into the next mat-mul's src1 (no copy in between)
        g.op_norm(x, 1e-5, rms=True, out=out)
    return Step("op_norm", shape, None, fn)


def chains(g, L, rng):
    import torch

    def w(t, M, K):
        return torch.from_numpy(O.random_blocks(t, M * K // R.qk(t), rng)).cuda()
    S0, GEMV = g.MM_SRC0_STATIC, g.MM_GEMV
    # n = 1: op_norm -> generic -> first-generation TMA -> superblock -> mma -> generic
    c1 = [norm_step(g, (1, 4096)),
          mm_step(g, O.Q4_K, w(O.Q4_K, 2048, 4096), 2048, 4096, 1, g.MM_GENERIC | S0, "generic"),
          mm_step(g, O.Q4_K, w(O.Q4_K, 4096, 2048), 4096, 2048, 1, GEMV | g.MM_GEMV_V1 | S0, "first-generation TMA"),
          mm_step(g, O.Q6_K, w(O.Q6_K, 11008, 4096), 11008, 4096, 1, GEMV | g.MM_GEMV_DP4A | S0, "superblock"),
          mm_step(g, O.Q4_K, w(O.Q4_K, 4096, 11008), 4096, 11008, 1, GEMV | g.MM_GEMV_MMA | S0, "mma"),
          mm_step(g, O.IQ2_XXS, w(O.IQ2_XXS, 1024, 4096), 1024, 4096, 1, g.MM_GENERIC | S0, "generic")]
    # n = 5: superblock -> mma -> wgmma -> op_norm -> generic -> superblock
    c2 = [mm_step(g, O.Q4_K, w(O.Q4_K, 4096, 4096), 4096, 4096, 5, GEMV | g.MM_GEMV_DP4A | S0, "superblock"),
          mm_step(g, O.Q5_0, w(O.Q5_0, 2048, 4096), 2048, 4096, 5, GEMV | g.MM_GEMV_MMA | S0, "mma"),
          mm_step(g, O.Q4_K, w(O.Q4_K, 4096, 2048), 4096, 2048, 5, g.MM_GEMM | S0, "wgmma"),
          norm_step(g, (5, 4096)),
          mm_step(g, O.Q8_0, w(O.Q8_0, 1024, 4096), 1024, 4096, 5, g.MM_GENERIC, "generic"),
          mm_step(g, O.Q4_K, w(O.Q4_K, 4096, 1024), 4096, 1024, 5, GEMV | g.MM_GEMV_DP4A, "superblock")]
    # n = 64: wgmma split-K -> dense -> mul_mat_f16 -> generic -> wgmma split-K (16 tiles, K = 512) -> wgmma split-K
    Wh = torch.from_numpy(rng.uniform(-0.05, 0.05, (2048, 1024)).astype(np.float16)).cuda()
    Wsk = w(O.Q8_0, 11008, 4096)
    c3 = [mm_step(g, O.Q8_0, Wsk, 11008, 4096, 64, g.MM_GEMM | S0, "wgmma", splitk=True),
          mm_step(g, O.IQ2_XXS, w(O.IQ2_XXS, 1024, 11008), 1024, 11008, 64, g.MM_GEMM | S0, "dense"),
          f16_step(L, g, Wh, 2048, 1024, 64),
          mm_step(g, O.Q4_0, w(O.Q4_0, 512, 2048), 512, 2048, 64, g.MM_GENERIC, "generic"),
          mm_step(g, O.Q4_K, w(O.Q4_K, 4096, 512), 4096, 512, 64, g.MM_GEMM, "wgmma", splitk=True),
          mm_step(g, O.Q8_0, Wsk, 11008, 4096, 64, g.MM_GEMM, "wgmma", splitk=True)]
    return [("n=1", c1, (1, 4096)), ("n=5", c2, (5, 4096)), ("n=64", c3, (64, 4096))]


def test_dependent_chains_bitwise(env):
    """every route family is a producer and a consumer in some chain (split-K wgmma too); each step's kernel is checked"""
    import torch
    g, L, orc = env
    rng = np.random.default_rng(7)
    ws = torch.full((256 << 20,), 0xFF, dtype=torch.uint8, device="cuda")
    for name, steps, xshape in chains(g, L, rng):
        for s in steps:
            if s.splitk is not None:                     # split-K shows in the workspace: partials beyond the fp16 copy and scales
                t, M, N, K = s.mm
                a = R.mm_args(L, t, M, N, K, g.MM_GEMM, 256)
                plain = ((N * K * 2 + 255) & ~255) + ((N * 4 + 255) & ~255) + 1024
                assert (int(L.ggml_b200_mul_mat_workspace_size(C.byref(a))) > plain) == s.splitk, s.name
        x0 = torch.from_numpy(rng.uniform(-1, 1, xshape).astype(np.float32)).cuda()
        a = run_chain(steps, x0, ws, sync=False)
        b = run_chain(steps, x0, ws, sync=True)
        for s, ya, yb in zip(steps, a, b):
            assert bool(torch.isfinite(yb).all()), f"chain {name}: {s.name} gave non-finite values with synchronisation"
            assert torch.equal(ya, yb), f"chain {name}: {s.name} differs from its synchronised run"


def test_independent_launch_between_dependent_pair(env):
    """A writes Y; B (SRC0 | SRC1_STATIC, fixed inputs) runs independently; C consumes Y: C must see all of A's Y (mmvq_sb.cu: a
    SRC1_STATIC launch waits for its predecessor before it retires, so completion stays transitive along the stream)"""
    import torch
    g, L, orc = env
    rng = np.random.default_rng(8)
    Wa = torch.from_numpy(O.random_blocks(O.Q4_K, 11008 * 4096 // 256, rng)).cuda()
    Wb = torch.from_numpy(O.random_blocks(O.Q4_K, 4096 * 4096 // 256, rng)).cuda()
    Wc = torch.from_numpy(O.random_blocks(O.Q6_K, 4096 * 11008 // 256, rng)).cuda()
    x = torch.from_numpy(rng.uniform(-1, 1, 4096).astype(np.float32)).cuda()
    xb = torch.from_numpy(rng.uniform(-1, 1, 4096).astype(np.float32)).cuda()
    ws = torch.full((64 << 20,), 0xFF, dtype=torch.uint8, device="cuda")
    S0, S1 = g.MM_SRC0_STATIC, g.MM_SRC1_STATIC
    res = []
    for sync in (False, True):
        ya = torch.full((11008,), float("nan"), device="cuda")
        yb = torch.full((4096,), float("nan"), device="cuda")
        yc = torch.full((4096,), float("nan"), device="cuda")
        torch.cuda.synchronize()
        for fn in (lambda: g.mul_mat(O.Q4_K, Wa, x, 11008, 1, 4096, flags=S0, out=ya.view(1, 1, 1, -1), workspace=ws),
                   lambda: g.mul_mat(O.Q4_K, Wb, xb, 4096, 1, 4096, flags=S0 | S1, out=yb.view(1, 1, 1, -1), workspace=ws),
                   lambda: g.mul_mat(O.Q6_K, Wc, ya, 4096, 1, 11008, flags=S0, out=yc.view(1, 1, 1, -1), workspace=ws)):
            fn()
            if sync:
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        res.append((ya.clone(), yb.clone(), yc.clone()))
    for u, v in zip(*res):
        assert bool(torch.isfinite(v).all()) and torch.equal(u, v)


# ---------------------------------------------------------------------------------------------------------------- large shapes
def need_free(nbytes: int):
    import torch
    free, total = torch.cuda.mem_get_info()
    if free < nbytes * 1.2:
        pytest.skip(f"needs {nbytes / 2**30:.1f} GiB free on the GPU, {free / 2**30:.1f} GiB of {total / 2**30:.1f} GiB are")


@pytest.mark.parametrize("t", [O.Q4_K, O.Q6_K], ids=["q4_K", "q6_K"])
def test_vocabulary_rows(t, env, report):
    """4096 -> 32000 at n = 1 (independent launch: more than 16 chunks per CTA take the atomic counter; default flags), 4 and 512"""
    import torch
    g, L, orc = env
    M, K = 32000, 4096
    need_free(M * K * 8 * 3 + (2 << 30))
    rng = np.random.default_rng(32000 + t)
    W = O.random_blocks(t, M * K // 256, rng)
    Wd = torch.from_numpy(W).cuda()
    ref = mm.Reference(orc, t, W, M, K, device="cuda")
    for N, flags in [(1, g.MM_SRC0_STATIC | g.MM_SRC1_STATIC), (1, 0), (4, g.MM_SRC0_STATIC), (512, g.MM_SRC0_STATIC)]:
        X = activations(rng, N, K)
        xt = torch.from_numpy(X).cuda()
        a = R.mm_args(L, t, M, N, K, flags, xt.data_ptr())
        a.src0 = Wd.data_ptr()
        ws_size = int(L.ggml_b200_mul_mat_workspace_size(C.byref(a)))

        def launch(outs, ws, a=a):
            a.dst, a.workspace, a.workspace_size = outs[0].data_ptr(), ptr(ws), ws.numel()
            g.check(L.ggml_b200_mul_mat(C.byref(a), stream()), "ggml_b200_mul_mat")
        what = f"{O.TYPE_NAMES[t]} {K}->{M} N={N} flags={flags}"
        (y,), _ = launch_twice(what, launch, [N * M], ws_size, [Wd, xt])
        y = y.view(N, M)
        kind = "f16" if N >= 9 else "int"
        check_values(what, y, *ref(X, kind), kind, report)


def test_output_over_2_31_bytes(env, report):
    """Q6_K 4096 -> 128256 at n = 4200: dst is 2.15 GB.  All rows of the last 32 and of 16 random columns, all columns of the first and
    last 256-row tiles, and every element finite (everything was written into the NaN-filled dst)"""
    import torch
    g, L, orc = env
    t, M, K, N = O.Q6_K, 128256, 4096, 4200
    need_free(N * M * 4 + M * K * 210 // 256 + N * K * 6 + 4 * 16384 * K * 8 + (2 << 30))
    rng = np.random.default_rng(128256)
    W = O.random_blocks(t, M * K // 256, rng)
    Wd = torch.from_numpy(W).cuda()
    X = activations(rng, N, K)
    xt = torch.from_numpy(X).cuda()
    a = R.mm_args(L, t, M, N, K, 0, xt.data_ptr())
    a.src0 = Wd.data_ptr()
    assert int(L.ggml_b200_mul_mat_plan(C.byref(a))) == g.MM_GEMM
    ws = Scratch(int(L.ggml_b200_mul_mat_workspace_size(C.byref(a)))).fill(0xFF)
    out = Poisoned(N * M).fill(float("nan"))
    a.dst, a.workspace, a.workspace_size = out.y.data_ptr(), ws.ws.data_ptr(), ws.n
    g.check(L.ggml_b200_mul_mat(C.byref(a), stream()), "ggml_b200_mul_mat")
    torch.cuda.synchronize()
    assert out.guards_ok() and ws.guards_ok()
    y = out.y.view(N, M)
    assert bool(torch.isfinite(y).all()), f"{int((~torch.isfinite(y)).sum())} elements not written"
    cols = np.concatenate([np.arange(N - 32, N), rng.choice(N - 32, 16, replace=False)])
    rb = 210 * K // 256
    for m0 in range(0, M, 16384):                        # all rows of the chosen columns, 16384 rows at a time
        m1 = min(M, m0 + 16384)
        ref = mm.Reference(orc, t, W[m0 * rb:m1 * rb], m1 - m0, K, device="cuda")
        r, bound = ref(X[cols], "f16")
        q = float(mm.ratio(y[torch.from_numpy(cols).cuda(), m0:m1], r, bound).max())
        assert q <= RATIO_GATE["f16"], (m0, q)
    for m0 in (0, M - 256):                              # all columns of the first and last tiles
        ref = mm.Reference(orc, t, W[m0 * rb:(m0 + 256) * rb], 256, K, device="cuda")
        check_values(f"q6_K 4096->128256 N=4200 rows {m0}..{m0 + 255}", y[:, m0:m0 + 256], *ref(X, "f16"), "f16", report)


def test_expert_stack_over_2_31_bytes(env, report):
    """per-pair MUL_MAT_ID over 256 experts x 2048 rows x K = 7424 Q4_K: 4176-byte rows, a 2.19e9-byte expert stack.  Tokens routed to
    experts 254 and 255, whose rows start past byte 2^31, and to low experts, into a poisoned dst and workspace"""
    import torch
    g, L, orc = env
    t, ne, nu, M, K, ntok = O.Q4_K, 256, 2, 2048, 7424, 4
    rb = 144 * K // 256
    assert ne * M * rb > 2 ** 31 and 254 * M * rb > 2 ** 31
    need_free(ne * M * rb + 2 * M * K * 8 + (1 << 30))
    gen = torch.Generator(device="cuda").manual_seed(255)
    Wd = torch.randint(0, 256, (ne * M * K // 256, 144), dtype=torch.uint8, device="cuda", generator=gen)
    Wd[:, 0:4] = (torch.rand(Wd.shape[0], 2, device="cuda", generator=gen) * (0.05 / 32)).half().view(torch.uint8)
    Wd = Wd.view(-1)
    rng = np.random.default_rng(255)
    X = activations(rng, ntok, K)
    xt = torch.from_numpy(X).cuda()
    ids = torch.tensor([[255, 254], [255, 0], [128, 255], [254, 1]], dtype=torch.int32, device="cuda")
    a = R.mmid_args(L, t, M, K, ne, nu, 1, ntok)
    ws_size = int(L.ggml_b200_mul_mat_id_workspace_size(C.byref(a)))

    def launch(outs, ws):
        g.mul_mat_id(t, Wd, xt, ids, M, K, ne, nu, 1, ntok, out=outs[0], workspace=ws)
    (y,), _ = launch_twice("mul_mat_id 256 x 2048 x 7424 q4_K", launch, [ntok * nu * M], ws_size, [xt, ids])
    y = y.view(ntok, nu, M)
    worst = 0.0
    for x in (255, 254, 128, 1, 0):
        W = Wd[x * M * rb:(x + 1) * M * rb].cpu().numpy()
        ref = mm.Reference(orc, t, W, M, K, device="cuda")
        for tok, e in zip(*np.nonzero(ids.cpu().numpy() == x)):
            r, bound = ref(X[tok][None], "int")
            worst = max(worst, float(mm.ratio(y[tok, e][None], r, bound).max()))
    report.append(("mul_mat_id 256 x 2048 x 7424 q4_K (2.19e9-byte stack)", "int", worst, 0.0, 0.0))
    assert worst <= RATIO_GATE["int"]


# ---------------------------------------------------------------------------------------------------------------- the worst values
@pytest.fixture(scope="module")
def report():
    rows = []
    yield rows
    if rows:
        for kind in ("int", "f16"):
            sel = [r for r in rows if r[1] == kind]
            if sel:
                w = max(sel, key=lambda r: r[2])
                print(f"\n{kind}: {len(sel)} cases, worst |y - r| / bound {w[2]:.3g} ({w[0]}), worst block NMSE {max(r[3] for r in sel):.3g}, "
                      f"worst column NMSE {max(r[4] for r in sel):.3g}")
