"""GPU: the small ops either side of every mat-mul (ops.cu get_rows_kernel, bin_bcast_kernel, norm_kernel, scale_kernel,
diag_mask_inf_kernel, unary_kernel, cpy_kernel and the fused norm_affine_kernel / soft_max_kernel), pinned to the f64 references of
oracle/core.py (which tests/test_oracle_core.py pins to ggml-cpu) and to ggml-cpu itself.  Gates are about 10 x the worst values measured
on an H100 (DESIGN.md §5).
  (a) through the C ABI against the references: GET_ROWS of every format bit-exact against Oracle.dequantize and the device's own
      dequantize (rows of 96 / 4128 / 256 / 4352, repeated / descending / batched ids, 3- and 4-dim src0, a padded dst); ADD / SUB / MUL /
      DIV bit-exact with broadcast along every subset of dims, permuted / transposed / padded / in-place operands, +-0 and subnormal
      divisors; NORM / RMS_NORM at row lengths either side of the launcher's 32 / 128 / 256-thread steps, no further from f64 than ggml-cpu
      on the same row; every unary function over finite values, +-0, +-inf, NaN and subnormals (bit-exact where it is one IEEE operation or
      ggml-cpu's f16 table, within the CUDA math library's ulp bound otherwise); SCALE and DIAG_MASK_INF bit-exact; float CPY / CONT / DUP
      bit-exact through permuted, transposed and padded views; a descriptor their checks refuse raises the check's code and launches nothing;
  (b) the same ops as graphs (oracle/core_probe.cpp) on B2000 against ggml-cpu, and the two chains the plug-in fuses (NORM -> MUL -> ADD,
      SCALE -> DIAG_MASK_INF -> SOFT_MAX), whose bits do not depend on the fusion and which run as one launch each."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import core as K
from oracle import decoder
from oracle import oracle as O
from oracle.pool import ES, F16, F32, Source

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]

# the CUDA math library's maximum error (CUDA C++ Programming Guide, "Mathematical Functions": expf, tanhf, sinf, cosf 2 ulp) plus one ulp
# for each rounding after it (SIGMOID: + and /; SILU: + and /).  Measured on an H100 80GB HBM3 at 700 W: SILU 2.26, TANH 1.72, SIGMOID
# 2.61, EXP 1.78, SIN 1.43, COS 1.42
DEVICE_ULP = {K.TANH: 2.0, K.EXP: 2.0, K.SIN: 2.0, K.COS: 2.0, K.SIGMOID: 4.0, K.SILU: 4.0}
# NORM / RMS_NORM sum in double and round as ggml-cpu does: measured, each row's NMSE against f64 equals ggml-cpu's (ratio 1.00; 2.8e-7 at
# worst, at offset 1e4, from rounding the mean to f32), and the plug-in's result is bit-identical to ggml-cpu's (NMSE 0)
NORM_CPU_RATIO = 2.0            # (a) a row's NMSE against f64 is at most this times ggml-cpu's on the same row ...
NORM_FLOOR = 1e-13              # ... or below f32 round-off (rows ggml-cpu gets exactly right)
NORM_CPU_NMSE = 1e-14           # (b) NORM / RMS_NORM and the fused chain on B2000 against ggml-cpu: a reordered double sum at most
SOFT_MAX_NMSE = 1.2e-13         # (b) the fused SCALE -> DIAG_MASK_INF -> SOFT_MAX against ggml-cpu: 8.7e-15 measured; test_gpu_attention's gate
# f16 inputs on which the device's GELU / GELU_QUICK (f32 tanhf / expf within 2 ulp, then rounded to f16) differ from ggml-cpu's table
# (measured on an H100: one for GELU, none for GELU_QUICK; ggml-cpu's table itself is what oracle/core.py computes, tests/test_oracle_core.py)
TABLE_EXCEPTIONS = {K.GELU: [-1.9990234375], K.GELU_QUICK: []}


@pytest.fixture(scope="module")
def plugin():
    return decoder.plugin("libggml_core_probe.so")


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def view(t, src: Source):
    """the torch view of a parent torch tensor that `src` describes"""
    ne, nb = src.view()
    es = ES[src.type]
    return t.as_strided(tuple(ne[::-1]), tuple(b // es for b in nb[::-1]), src.offs // es)


def host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


# ------------------------------------------------------------------ (a) GET_ROWS
@pytest.mark.parametrize("case", K.get_rows_grid(), ids=lambda c: f"{O.TYPE_NAMES[c[0].type]}-{c[0].ne}-{c[2]}")
def test_get_rows_c_abi_is_bit_exact(case):
    import torch
    import ggml_b200 as g
    src, n, order = case
    parent = K.get_rows_parent(src)
    ids = K.get_rows_ids(n, src.ne[2], src.ne[3], src.ne[1], order, src.seed)
    ne0 = src.ne[0]
    buf = dev(parent)
    nb0 = ES[src.type] if src.type in ES else K.row_bytes(src.type, K.orc().blck_size(src.type))        # one element / one block
    d = g.bytes_desc(buf, src.type, src.ne, (nb0,) + src.nb)
    padded = torch.full(ids.shape + (ne0 + 7,), float("nan"), dtype=torch.float32, device="cuda")     # a dst row stride past ne0
    got = host(g.op_get_rows(d, dev(ids), padded[..., :ne0]))
    want = K.get_rows_reference(src, parent, ids)
    assert K.same_bits(got, want).all(), (O.TYPE_NAMES[src.type], int((~K.same_bits(got, want)).sum()))
    assert np.isnan(host(padded)[..., ne0:]).all()                                                  # the padding is untouched
    if src.type not in (F32, F16):
        all_rows = host(g.dequantize(src.type, buf, int(np.prod(src.parent_ne)))).reshape(src.parent_ne[::-1])
        sel = np.stack([[all_rows[i12, i11, ids[i12, i11]] for i11 in range(ids.shape[1])] for i12 in range(ids.shape[0])])
        assert K.same_bits(got, sel).all()


# ------------------------------------------------------------------ (a) ADD / SUB / MUL / DIV
@pytest.mark.parametrize("case", K.binary_grid(), ids=lambda c: f"{K.BIN_NAMES[c[0]]}-{c[1].ne}{'T' * c[1].transpose}-{c[2].ne}"
                         f"{'-inplace' * c[3]}")
def test_binary_c_abi_is_bit_exact(case):
    import ggml_b200 as g
    op, s0, s1, inplace, _ = case
    p0, p1 = K.binary_values(s0), K.binary_values(s1)
    t0, t1 = dev(p0), dev(p1)
    a, b = view(t0, s0), view(t1, s1)
    want = K.binary_reference(op, K.logical(s0, p0), K.logical(s1, p1))
    got = host(g.op_bin_bcast(op, a, b, out=a if inplace else None))
    assert K.same_bits(got, want).all(), int((~K.same_bits(got, want)).sum())
    if inplace:                                                     # the padding of src0's rows is untouched
        assert K.same_bits(host(t0)[..., s0.ne[0]:], p0[..., s0.ne[0]:]).all()


# ------------------------------------------------------------------ (a) NORM / RMS_NORM
_norm_stats = {"ratio": 0.0, "nmse": 0.0}


@pytest.mark.parametrize("case", K.norm_grid(), ids=lambda c: f"{'rms' if c[0] else 'norm'}-{c[2].ne}-eps{c[1]:g}-off{c[3]:g}{'-zeros' * c[4]}")
def test_norm_c_abi_is_as_close_to_f64_as_ggml_cpu(plugin, case):
    import ggml_b200 as g
    rms, eps, src, offset, zero_rows = case
    parent = K.norm_values(src.parent_ne, offset, src.seed, zero_rows)
    x = K.logical(src, parent)
    got = host(g.op_norm(view(dev(parent), src), eps, rms)).reshape(-1, src.ne[0])
    cpu = K.norm("CPU", rms, eps, src, parent).reshape(-1, src.ne[0])
    exact = K.norm_reference(x, eps, rms, f32_mean=False).reshape(-1, src.ne[0])
    assert (np.isnan(got) == np.isnan(cpu)).all()
    for r in range(got.shape[0]):
        if np.isnan(cpu[r]).any():
            continue
        e_dev, e_cpu = K.nmse64(got[r], exact[r]), K.nmse64(cpu[r], exact[r])
        _norm_stats["nmse"] = max(_norm_stats["nmse"], e_dev)
        if e_cpu > 0:
            _norm_stats["ratio"] = max(_norm_stats["ratio"], e_dev / e_cpu)
        assert e_dev <= max(NORM_CPU_RATIO * e_cpu, NORM_FLOOR), (r, e_dev, e_cpu)
    print(f"NORM worst so far: NMSE vs f64 {_norm_stats['nmse']:.2e}, ratio to ggml-cpu {_norm_stats['ratio']:.2f}")


# ------------------------------------------------------------------ (a) unary, SCALE, DIAG_MASK_INF
def table_mismatches(op, got, want, x):
    bad = ~K.same_bits(got, want)
    # every disagreement is one f16 step: the two f32 results straddled a rounding boundary
    with np.errstate(over="ignore"):
        steps = [v.astype(np.float16).view(np.int16).astype(np.int64) for v in (got[bad], want[bad])]
    ulps = np.abs(steps[0] - steps[1])
    assert (ulps <= 1).all(), (K.UNARY_NAMES[op], x[bad][ulps > 1][:8])
    return sorted(float(v) for v in x[bad])


@pytest.mark.parametrize("op", range(14), ids=lambda o: K.UNARY_NAMES[o])
def test_unary_c_abi_against_the_reference(op):
    import ggml_b200 as g
    x = K.f16_inputs() if op in K.TABLE_UNARY else K.unary_values(op, 1 << 16)
    got = host(g.op_unary(op, dev(x)))
    ref = K.unary_reference(op, x)
    if op in K.EXACT_UNARY:
        bad = ~K.same_bits(got, ref)
        assert not bad.any(), (x[bad][:8], got[bad][:8], ref[bad][:8])
    elif op in K.TABLE_UNARY:
        mism = table_mismatches(op, got, ref, x)
        print(f"{K.UNARY_NAMES[op]}: {len(mism)} f16 inputs differ from ggml-cpu's table: {mism}")
        assert mism == TABLE_EXCEPTIONS[op]
    else:
        e = K.ulp_error(got, ref, K.SILU_TINY if op == K.SILU else K.FLT_MIN)
        print(f"{K.UNARY_NAMES[op]}: worst {e.max():.3f} ulp at x = {x[np.argmax(e)]!r}")
        assert e.max() <= DEVICE_ULP[op], (float(e.max()), float(x[np.argmax(e)]))


def test_gelu_quick_follows_the_f16_table_at_its_edges():
    import ggml_b200 as g
    x = np.array([65519.0, 65520.0, 1e6, np.inf, -65519.0, -65520.0, -np.inf, np.nan, -0.0, 3e-8], np.float32)
    got = host(g.op_unary(K.GELU_QUICK, dev(x)))
    assert got[0] == 65504.0 and np.isposinf(got[1:4]).all() and got[4] == 0.0 and np.isnan(got[5:8]).all()
    assert K.same_bits(got, K.gelu_quick_table(x)).all()


def test_scale_and_diag_mask_inf_c_abi_are_exact():
    import ggml_b200 as g
    x = K.binary_values(Source(F32, (37, 9, 4, 2), seed=3))
    for scale, n_past in ((0.125, 0), (-3.7, 5), (1e-30, 40)):
        s = host(g.op_scale(dev(x), scale))
        want_s = (x.astype(np.float64) * np.float32(scale)).astype(np.float32)
        assert K.same_bits(s, want_s).all()
        m = host(g.op_diag_mask_inf(dev(want_s), n_past))
        i1, i0 = np.arange(9)[:, None], np.arange(37)[None, :]
        assert K.same_bits(m, np.where(i0 > n_past + i1, -np.inf, want_s)).all()


def test_descriptor_launchers_refuse_what_their_checks_refuse():
    """SCALE, DIAG_MASK_INF, the unary ops, SOFT_MAX and the fused norm: one bad descriptor each gives its check's code and launches nothing"""
    import torch
    import ggml_b200 as g
    x = torch.randn(3, 9, 37, device="cuda")
    v = torch.randn(37, device="cuda")
    bad = [(lambda: g.op_scale(x.half(), 0.5), -1),                                 # f16 src
           (lambda: g.op_diag_mask_inf(x.transpose(1, 2), 0), -1),                  # transposed src
           (lambda: g.op_unary(14, x), -2),                                         # no such function
           (lambda: g.op_soft_max(x, mask=torch.zeros(9, 36, device="cuda")), -2),  # mask narrower than ne0
           (lambda: g.op_norm_affine(x, v[:36], v, 1e-5), -2)]                      # gain of ne0 - 1
    for i, (launch, code) in enumerate(bad):
        n0 = g.launch_count()
        with pytest.raises(g.B200Error, match=rf"failed \({code}\)"):
            launch()
        assert g.launch_count() == n0, i
    torch.cuda.synchronize()


# ------------------------------------------------------------------ (a) float CPY / CONT / DUP
@pytest.mark.parametrize("case", K.cpy_grid(), ids=lambda c: f"{('cpy', 'cont', 'dup')[c[0]]}-{c[1].type}-{c[1].ne}{'T' * c[1].transpose}")
def test_float_cpy_c_abi_is_bit_exact(case):
    import torch
    import ggml_b200 as g
    op, src, dst = case
    parent = K.cpy_values(src)
    s = view(dev(parent), src)
    if op == 0:
        dst_in = K.cpy_dst_in(dst)
        td = dev(dst_in)
        g.op_cpy(s, view(td, dst))
        got, want = host(td), K.cpy_expected(src, parent, dst, dst_in)
    else:                                                           # CONT / DUP: a copy into a packed tensor of the source's type
        y = torch.empty(tuple(src.view()[0][::-1]), dtype=s.dtype, device="cuda")
        g.op_cpy(s, y)
        got, want = host(y), K.cpy_reference(K.logical(src, parent), src.type)
    assert K.same_bits(got, want).all(), int((~K.same_bits(got, want)).sum())


# ------------------------------------------------------------------ (b) the plug-in against ggml-cpu
def test_get_rows_graph_matches_ggml_cpu(plugin):
    for src, n, order in K.get_rows_grid():
        parent = K.get_rows_parent(src)
        ids = K.get_rows_ids(n, src.ne[2], src.ne[3], src.ne[1], order, src.seed)
        assert K.same_bits(K.get_rows("B2000", src, parent, ids), K.get_rows("CPU", src, parent, ids)).all(), O.TYPE_NAMES[src.type]


def test_binary_graph_matches_ggml_cpu(plugin):
    for op, s0, s1, inplace, cpu_can in K.binary_grid():
        if not cpu_can:
            continue
        p0, p1 = K.binary_values(s0), K.binary_values(s1)
        assert K.same_bits(K.binary("B2000", op, s0, p0, s1, p1, inplace), K.binary("CPU", op, s0, p0, s1, p1, inplace)).all(), (op, s0, s1)


def test_norm_graph_matches_ggml_cpu(plugin):
    worst = 0.0
    for rms, eps, src, offset, zero_rows in K.norm_grid():
        parent = K.norm_values(src.parent_ne, offset, src.seed, zero_rows)
        got, cpu = K.norm("B2000", rms, eps, src, parent), K.norm("CPU", rms, eps, src, parent)
        nan = np.isnan(cpu)
        assert (np.isnan(got) == nan).all()
        e = K.nmse64(got[~nan], cpu[~nan])
        worst = max(worst, e)
        assert e <= NORM_CPU_NMSE, (rms, eps, src.ne, offset, e)
    print(f"NORM / RMS_NORM B2000 vs ggml-cpu: worst NMSE {worst:.2e}")


@pytest.mark.parametrize("op", range(14), ids=lambda o: K.UNARY_NAMES[o])
def test_unary_graph_matches_ggml_cpu(plugin, op):
    x = K.f16_inputs() if op in K.TABLE_UNARY else K.unary_values(op, 1 << 14)
    got, cpu = K.unary("B2000", op, x), K.unary("CPU", op, x)
    if op in K.EXACT_UNARY:
        assert K.same_bits(got, cpu).all()
    elif op in K.TABLE_UNARY:
        assert table_mismatches(op, got, cpu, x) == TABLE_EXCEPTIONS[op]
    else:                                   # both within their bounds of f64
        e = K.ulp_error(got, K.unary_reference(op, x), K.SILU_TINY if op == K.SILU else K.FLT_MIN)
        assert e.max() <= DEVICE_ULP[op], (float(e.max()), float(x[np.argmax(e)]))


def test_scale_mask_and_cpy_graphs_match_ggml_cpu(plugin):
    x = K.binary_values(Source(F32, (37, 9, 4, 2), seed=4))
    for scale, n_past in ((0.125, 0), (-3.7, 5)):
        for a, b in zip(K.scale_mask("B2000", x, scale, n_past), K.scale_mask("CPU", x, scale, n_past)):
            assert K.same_bits(a, b).all()
    for op, src, dst in K.cpy_grid():
        parent = K.cpy_values(src)
        dst_in = None if dst is None else K.cpy_dst_in(dst)
        assert K.same_bits(K.cpy("B2000", op, src, parent, dst, dst_in), K.cpy("CPU", op, src, parent, dst, dst_in)).all(), (op, src)


def fused_chain_cases():
    rng = np.random.default_rng(31)
    out = []
    for k, (ne0, rows) in enumerate(((768, 7), (4096, 3), (33, 5), (14336, 2))):
        x = (rng.standard_normal((1, 2, rows, ne0)) + (0.0, 30.0)[k % 2]).astype(np.float32)
        out.append((k % 2 == 1, 1e-5, x, rng.standard_normal(ne0).astype(np.float32), rng.standard_normal(ne0).astype(np.float32)))
    return out


def softmax_chain_cases():
    rng = np.random.default_rng(32)
    return [((rng.standard_normal(s) * 3.0).astype(np.float32), scale, n_past)
            for s, scale, n_past in (((1, 12, 7, 7), 0.125, 0), ((2, 4, 5, 69), 0.0883883, 64), ((1, 2, 3, 1500), 1.0, 1497))]


def plugin_launch_count() -> int:
    """the kernels the plug-in loaded into the reference has launched so far (its ggml_backend_b200_launch_count, found through the registry)"""
    import ctypes as C
    ggml = C.CDLL(str(O.REF_DIR / "libggml.so"))
    ggml.ggml_backend_reg_by_name.restype, ggml.ggml_backend_reg_by_name.argtypes = C.c_void_p, [C.c_char_p]
    ggml.ggml_backend_reg_get_proc_address.restype, ggml.ggml_backend_reg_get_proc_address.argtypes = C.c_void_p, [C.c_void_p, C.c_char_p]
    fn = ggml.ggml_backend_reg_get_proc_address(ggml.ggml_backend_reg_by_name(b"B200"), b"ggml_backend_b200_launch_count")
    assert fn
    return int(C.CFUNCTYPE(C.c_uint64)(fn)())


def run_fused_chains(dev_name):
    """every output of the two chains on `dev_name`, in one list, and the plug-in's kernel launches for each chain (the probe graphs have
    fewer than 8 nodes, so they run eagerly and every launch is counted)"""
    out, launches = [], []

    def counted(probe, *args):
        n0 = plugin_launch_count()
        r = probe(dev_name, *args)
        launches.append(plugin_launch_count() - n0)
        return r
    for rms, eps, x, gain, bias in fused_chain_cases():
        out += list(counted(K.norm_affine, rms, eps, x, gain, bias))
    for x, scale, n_past in softmax_chain_cases():
        out.append(counted(K.scale_mask_softmax, x, scale, n_past))
    return out, launches


def test_fused_chains_match_ggml_cpu_and_the_unfused_nodes(plugin, tmp_path):
    (got, launches), (cpu, _) = run_fused_chains("B2000"), run_fused_chains("CPU")
    n_norm = 3 * len(fused_chain_cases())
    worst_n = max(K.nmse64(a, b) for a, b in zip(got[:n_norm], cpu[:n_norm]))
    worst_s = max(K.nmse64(a, b) for a, b in zip(got[n_norm:], cpu[n_norm:]))
    print(f"fused chains B2000 vs ggml-cpu: NORM -> MUL -> ADD worst NMSE {worst_n:.2e}, SCALE -> DIAG_MASK_INF -> SOFT_MAX {worst_s:.2e}")
    assert worst_n <= NORM_CPU_NMSE and worst_s <= SOFT_MAX_NMSE
    # the same graphs with fusion disabled (read once per process: a fresh interpreter)
    script = ("import sys, numpy as np; sys.path[:0] = [sys.argv[1], sys.argv[1] + '/tests']; from oracle import decoder; "
              "from test_gpu_core_ops import run_fused_chains; decoder.plugin('libggml_core_probe.so'); "
              "out, launches = run_fused_chains('B2000'); np.savez(sys.argv[2], *out, launches=launches)")
    env = dict(os.environ, GGML_B200_DISABLE_FUSION="1")
    p = subprocess.run([sys.executable, "-c", script, str(ROOT), str(tmp_path / "unfused.npz")], env=env, capture_output=True, text=True,
                       timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    unfused = np.load(tmp_path / "unfused.npz")
    for i, a in enumerate(got):
        assert K.same_bits(a, unfused[f"arr_{i}"]).all(), i
    # each chain ran as one launch instead of three: a chain the plug-in stopped fusing would still pass on bits
    assert [u - 2 for u in unfused["launches"]] == launches, (launches, list(unfused["launches"]))
