"""GPU: the attention path's kernels every decoder runs each token (ops.cu flash_attn_ext_kernel, soft_max_kernel, cpy_kernel /
cpy_f32_q_kernel and mul_mat_f_kernel), pinned to the f64 references of oracle/attn.py (which tests/test_oracle_attn.py pins to ggml-cpu)
and to ggml-cpu itself.  Gates are about 10 x the worst values measured on an H100 (DESIGN.md §5).
  (a) FLASH_ATTN_EXT through the C ABI against f64 of the values it reads: every K / V format (f32 and f16 at D 40..256, the 32-element
      formats at D 64 / 128, the 256-element ones at D 256, K != V), GQA 32:32 / 32:8 / 32:1, ALiBi at 12 and 20 heads, causal and finite
      masks, softcap 30, n_kv 1..4099, n_q 1 / 7 / 64, ne3 2 over one K / V, K / V as views of a cache, Q permuted; bitwise repeatable,
      and each query row of an n_q launch equal to its own n_q = 1 launch;
  (b) FLASH_ATTN_EXT and SOFT_MAX as one-node graphs (oracle/attn_probe.cpp) on B2000 against ggml-cpu: the plug-in's binding of
      descriptors and op_params;
  (c) SOFT_MAX through the C ABI against f64: row lengths either side of the launcher's thread-count steps, f16 / f32 masks with more rows
      than the input, ALiBi at 1..48 heads, in place;
  (d) CPY bit-exact: f32 -> Q8_0 (ties to even, as ggml-cpu writes it on x86), Q4_0 and f16 into views of caches at an offset, from packed,
      padded and permuted sources, through the C ABI and the plug-in; f16 -> f32;
  (e) the float MUL_MAT through the C ABI against f64 of the operands it reads."""
from pathlib import Path

import numpy as np
import pytest

from oracle import attn as A
from oracle import decoder
from oracle import oracle as O
from oracle.pool import F16, F32, Source

pytestmark = pytest.mark.gpu
G_DIR = Path(__file__).resolve().parent / "golden"

# measured worsts on an H100 80GB HBM3 at 700 W: (a) 3.1e-13 (f32 K / V; 1e-14 .. 3e-13 over the block formats); (b) FA 1.4e-4 (iq2_xs and
# iq1_s), SOFT_MAX 1.2e-14; (c) 1.2e-14; (e) 7.6e-15
FA_NMSE = 3e-12                 # (a)
FA_CPU_NMSE = 5e-4              # (b): the reference's own FA gate (ggml-cpu quantizes Q to K's vec-dot type, accumulates an f16 V in f16)
SOFT_MAX_NMSE = 1.2e-13         # (b), (c)
MUL_MAT_NMSE = 8e-14            # (e)


@pytest.fixture(scope="module")
def plugin():
    return decoder.plugin("libggml_attn_probe.so")


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------ (a) FLASH_ATTN_EXT through the C ABI
def fa_grid():
    """axes to cover rather than their product; every K / V type appears with GQA and a mask"""
    out, seed = [], 100
    heads = [(32, 32), (32, 8), (32, 1)]
    D_FLOAT = (40, 64, 80, 96, 112, 128, 256)
    for i, D in enumerate(D_FLOAT):
        for j, t in enumerate((F32, F16)):
            k = 2 * i + j
            h, hk = heads[k % 3]
            out.append(A.FaCase(D, (1, 3, 5, 127, 1024, 4099)[k % 6], (1, 7, 64)[k % 3], h, hk, t, t, ne3=1 + k % 2,
                                mask=("causal", "finite")[k % 2], softcap=30.0 if k % 4 == 1 else 0.0, permute_q=k % 3 == 2, seed=seed))
            seed += 1
    for i, t in enumerate(A.BLOCK_TYPES_32):
        for j, D in enumerate((64, 128)):
            k = 2 * i + j
            h, hk = heads[1 + k % 2]
            out.append(A.FaCase(D, (127, 5, 1024, 3)[k % 4], (7, 1, 64)[k % 3], h, hk, t, t, ne3=1 + k % 2,
                                mask=("finite", "causal")[k % 2], softcap=30.0 if k % 5 == 2 else 0.0, permute_q=k % 2 == 1, seed=seed))
            seed += 1
    for i, t in enumerate(A.BLOCK_TYPES_256):
        h, hk = heads[1 + i % 2]
        out.append(A.FaCase(256, (4099 if i < 2 else (127, 1024, 5)[i % 3]), (1, 7)[i % 2], h, hk, t, t, ne3=1 + i % 2,
                            mask=("causal", "finite")[i % 2], softcap=30.0 if i % 4 == 3 else 0.0, permute_q=i % 3 == 0, seed=seed))
        seed += 1
    out += [A.FaCase(128, 300, 7, 32, 8, F16, O.Q8_0, mask="causal", seed=seed),                 # K != V
            A.FaCase(256, 260, 3, 32, 8, O.Q4_K, O.Q6_K, mask="finite", permute_q=True, seed=seed + 1),
            A.FaCase(64, 127, 7, 12, 12, F16, F16, mask="finite", max_bias=8.0, seed=seed + 2),      # ALiBi, both slope branches
            A.FaCase(128, 1024, 7, 20, 4, O.Q8_0, O.Q8_0, mask="finite", max_bias=8.0, ne3=2, seed=seed + 3),
            A.FaCase(96, 129, 64, 20, 20, F32, F32, mask="finite", max_bias=8.0, softcap=30.0, permute_q=True, seed=seed + 4),
            A.FaCase(80, 33, 7, 32, 8, F16, F16, seed=seed + 5)]                                   # no mask
    return out


def fa_device(case, d, q_rows=None):
    """FLASH_ATTN_EXT of `case` through the C ABI, K and V read through bytes_desc views of the uploaded caches (q_rows: a slice of the
    query rows, with the matching mask rows)"""
    import ggml_b200 as g
    qp = dev(d.q_parent)
    q = qp.permute(0, 2, 1, 3) if case.permute_q else qp
    mask = None if d.mask is None else dev(d.mask)
    if q_rows is not None:
        q = q[:, :, q_rows]
        mask = None if mask is None else mask[q_rows]
    kc, vc = dev(d.k_cache), dev(d.v_cache)
    descs = []
    for t, buf in ((case.kt, kc), (case.vt, vc)):
        s = case.kv_source(t)
        nb0 = A.row_bytes(t, 1 if t in (F32, F16) else A.orc().blck_size(t))          # one element or one block
        descs.append(g.bytes_desc(buf, t, s.ne, (nb0,) + tuple(s.nb)))
    return g.op_flash_attn_ext(q, descs[0], descs[1], mask, d.scale, case.max_bias, case.softcap)


def test_flash_attn_c_abi_matches_f64():
    import torch
    worst, per_type = 0.0, {}
    for case in fa_grid():
        d = A.fa_data(case)
        got = fa_device(case, d)
        torch.cuda.synchronize()
        got = got.cpu().numpy()
        assert np.isfinite(got).all(), str(case)
        e = O.nmse(got, A.flash_attn_reference(case, d))
        name = f"{O.TYPE_NAMES[case.kt]}/{O.TYPE_NAMES[case.vt]}"
        per_type[name] = max(per_type.get(name, 0.0), e)
        worst = max(worst, e)
        assert e <= FA_NMSE, (str(case), e)
    print(f"FLASH_ATTN_EXT C ABI vs f64: {len(fa_grid())} cases, worst NMSE {worst:.2e}; per K/V type: "
          + ", ".join(f"{k} {v:.1e}" for k, v in sorted(per_type.items())))


def test_flash_attn_is_repeatable_and_row_independent():
    import torch
    for case in (A.FaCase(128, 1024, 64, 32, 8, O.Q4_0, O.Q4_0, mask="causal", permute_q=True, seed=900),
                 A.FaCase(96, 127, 7, 20, 20, F16, F16, mask="finite", max_bias=8.0, softcap=30.0, seed=901)):
        d = A.fa_data(case)
        a, b = fa_device(case, d), fa_device(case, d)
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), str(case)
        for i in range(case.n_q):
            one = fa_device(case, d, slice(i, i + 1))
            assert torch.equal(one.view(torch.int32), a[:, i: i + 1].view(torch.int32)), (str(case), i)


# ------------------------------------------------------------------ (b) one-node graphs on B2000 against ggml-cpu
def fa_probe_grid():
    """one case per K / V type ggml-cpu runs (it aborts on an f32 K), each with GQA and a mask, plus ALiBi, softcap, K != V and permuted Q"""
    out = []
    for i, t in enumerate((F16,) + A.BLOCK_TYPES_32 + A.BLOCK_TYPES_256):
        D = 256 if t in A.BLOCK_TYPES_256 else (64, 128)[i % 2]
        out.append(A.FaCase(D, (77, 130, 33)[i % 3], (3, 7)[i % 2], 32, (8, 1)[i % 2], t, t, ne3=1 + i % 2, mask=("causal", "finite")[i % 2],
                            permute_q=i % 3 == 0, seed=1000 + i))
    out += [A.FaCase(64, 50, 4, 12, 12, F16, F16, mask="finite", max_bias=8.0, seed=1100),
            A.FaCase(64, 50, 4, 20, 4, O.Q4_0, O.Q4_0, mask="finite", max_bias=8.0, seed=1101),
            A.FaCase(64, 33, 2, 8, 8, F16, F16, mask="causal", softcap=30.0, seed=1102),
            A.FaCase(64, 29, 7, 4, 4, F16, O.Q8_0, mask="causal", seed=1103),
            A.FaCase(256, 19, 3, 4, 2, O.Q4_K, O.Q6_K, mask="finite", ne3=2, seed=1104)]
    return out


def test_flash_attn_graph_matches_ggml_cpu(plugin):
    per_type = {}
    for case in fa_probe_grid():
        d = A.fa_data(case)
        got, want = A.flash_attn_ext("B2000", case, d), A.flash_attn_ext("CPU", case, d)
        e = O.nmse(got, want)
        assert e <= FA_CPU_NMSE, (str(case), e)
        name = f"{O.TYPE_NAMES[case.kt]}/{O.TYPE_NAMES[case.vt]}"
        per_type[name] = max(per_type.get(name, 0.0), e)
    print("FLASH_ATTN_EXT B2000 vs ggml-cpu, worst NMSE per K/V type: " + ", ".join(f"{k} {v:.1e}" for k, v in sorted(per_type.items())))


SOFT_MAX_PROBE_CASES = [A.SoftMaxCase((33, 4, 5, 1), F16, 8, scale=0.5, max_bias=8.0, seed=1),
                        A.SoftMaxCase((129, 3, 12, 2), F32, 4, scale=0.125, max_bias=8.0, seed=2),
                        A.SoftMaxCase((1025, 2, 3, 1), F16, 64, scale=1.0, seed=3),
                        A.SoftMaxCase((4096, 7, 32, 1), F16, 64, scale=0.0625, seed=4),
                        A.SoftMaxCase((32, 5, 1, 1), scale=2.0, seed=5)]


def test_soft_max_graph_matches_ggml_cpu(plugin):
    worst = 0.0
    for case in SOFT_MAX_PROBE_CASES:
        data = A.soft_max_data(case)
        e = O.nmse(A.soft_max("B2000", case, data), A.soft_max("CPU", case, data))
        assert e <= SOFT_MAX_NMSE, (str(case), e)
        worst = max(worst, e)
    print(f"SOFT_MAX B2000 vs ggml-cpu: worst NMSE {worst:.2e}")


# ------------------------------------------------------------------ (c) SOFT_MAX through the C ABI
def soft_max_grid():
    out = []
    heads = (1, 5, 12, 32, 48)
    for i, ne0 in enumerate((1, 31, 32, 33, 127, 128, 129, 1023, 1024, 1025, 4096, 32000)):
        h = heads[i % 5] if ne0 < 32000 else 5
        out.append(A.SoftMaxCase((ne0, 3, h, 1 + i % 2), (F16, F32)[i % 2], 3 + 2 * (i % 3), scale=(1.0, 0.125)[i % 2],
                                 max_bias=(0.0, 8.0)[(i // 2) % 2], seed=200 + i))
    out += [A.SoftMaxCase((200, 4, h, 1), F16, 7, scale=0.5, max_bias=8.0, seed=220 + h) for h in heads]
    out += [A.SoftMaxCase((513, 3, 2, 2), scale=0.25, seed=240)]
    return out


def test_soft_max_c_abi_matches_f64():
    import torch
    import ggml_b200 as g
    worst = 0.0
    for inplace in (False, True):
        for case in soft_max_grid():
            x, mask = A.soft_max_data(case)
            xt = dev(x)
            y = g.op_soft_max(xt, case.scale, mask=None if mask is None else dev(mask), max_bias=case.max_bias, inplace=inplace)
            torch.cuda.synchronize()
            assert (y.data_ptr() == xt.data_ptr()) == inplace
            e = O.nmse(y.cpu().numpy(), A.soft_max_reference(case, x, mask))
            assert e <= SOFT_MAX_NMSE, (str(case), inplace, e)
            worst = max(worst, e)
    print(f"SOFT_MAX C ABI vs f64: {2 * len(soft_max_grid())} cases, worst NMSE {worst:.2e}")


# ------------------------------------------------------------------ (d) CPY, bit-exact
def cpy_device(case, parent, cache):
    import torch
    import ggml_b200 as g
    pt, ct = dev(parent.view(np.uint8).reshape(-1)), dev(cache)
    ne, nb = case.src.view()
    s = g.bytes_desc(pt, F32, ne, nb, case.src.offs)
    ds = case.dst_source()
    nb0 = 2 if case.dst_type == F16 else A.row_bytes(case.dst_type, 32)
    g.op_cpy(s, g.bytes_desc(ct, case.dst_type, ds.ne, (nb0,) + tuple(ds.nb), ds.offs))
    torch.cuda.synchronize()
    return ct.cpu().numpy()


def test_cpy_into_a_cache_is_bit_exact(plugin):
    gx = np.load(G_DIR / "act_q8.npz")["x"]
    for case in A.cpy_grid():
        parent, cache = A.cpy_parent(case, gx), A.cache_in(case)
        want = A.cpy_expected(case, parent, cache)
        assert np.array_equal(cpy_device(case, parent, cache), want), f"C ABI: {case}"
        assert np.array_equal(A.cpy("B2000", case, parent, cache), want), f"B2000: {case}"
        assert np.array_equal(A.cpy("CPU", case, parent, cache), want), f"CPU: {case}"


def test_cpy_q8_0_rounds_ties_to_even():
    """the Q8_0 cache ggml-cpu writes: on half-integer codes the _ref rounding (away from zero) gives other bytes"""
    case = A.CpyCase(Source(F32, (256, 64), seed=300), O.Q8_0, (256, 64), 70, 3, "ties")
    parent, cache = A.cpy_parent(case), A.cache_in(case)
    got, want = cpy_device(case, parent, cache), A.cpy_expected(case, parent, cache)
    assert np.array_equal(got, want), f"{int((got != want).sum())} of {got.size} cache bytes differ from ggml-cpu's"


def test_cpy_f16_to_f32_and_back():
    import torch
    import ggml_b200 as g
    h = np.random.default_rng(310).integers(0, 1 << 16, 4096, dtype=np.uint64).astype(np.uint16)
    h[(h & 0x7C00) == 0x7C00] = 0x3C00                               # no NaN / inf: those words are compared by value below
    ht = dev(h.view(np.float16).reshape(64, 64))
    f = torch.empty((64, 64), dtype=torch.float32, device="cuda")
    g.op_cpy(ht, f)
    x = np.random.default_rng(311).standard_normal((33, 64)).astype(np.float32) * np.float32(3000.0)
    back = torch.empty((64, 33), dtype=torch.float16, device="cuda")
    g.op_cpy(dev(x), back.t())                                        # into a transposed view
    torch.cuda.synchronize()
    assert np.array_equal(f.cpu().numpy(), h.view(np.float16).reshape(64, 64).astype(np.float32))
    assert np.array_equal(back.t().cpu().numpy().view(np.uint16), x.astype(np.float16).view(np.uint16))


# ------------------------------------------------------------------ (e) the float MUL_MAT through the C ABI
def test_mul_mat_f_c_abi_matches_f64():
    import torch
    import ggml_b200 as g
    rng = np.random.default_rng(400)
    r = lambda *shape: torch.from_numpy(rng.standard_normal(shape).astype(np.float32)).cuda()
    V = r(4, 300, 96)                                                  # [n_head, n_kv, D]: V^T is a view with nb0 = a whole row
    Kc = r(6, 2, 129)                                                  # [n_tok, n_head, K]: read permuted as [n_head, n_tok, K]
    cases = [("f32 x f32", r(2, 3, 70, 129), r(2, 3, 5, 129)),
             ("f16 x f16", r(2, 3, 70, 129).half(), r(2, 3, 5, 129).half()),
             ("f16 x f32", r(3, 40, 257).half(), r(3, 9, 257)),
             ("broadcast 4:1", r(1, 2, 33, 64), r(1, 8, 7, 64)),
             ("permuted src1", r(2, 50, 129), Kc.permute(1, 0, 2)),
             ("transposed V", V.transpose(1, 2), r(4, 7, 300)),
             ("transposed f16 V", V.half().transpose(1, 2), r(4, 7, 300))]
    worst = 0.0
    for name, a, b in cases:
        y = g.op_mul_mat_f(a, b)
        torch.cuda.synchronize()
        a64 = a.double()
        b64 = b.half().double() if (a.dtype == torch.float16 and b.dtype == torch.float32) else b.double()   # what the kernel reads
        a64 = a64.repeat_interleave(b.shape[-3] // a.shape[-3], dim=-3) if a.dim() >= 3 else a64
        want = (b64 @ a64.transpose(-1, -2)).cpu().numpy()
        e = O.nmse(y.cpu().numpy(), want)
        assert e <= MUL_MAT_NMSE, (name, e)
        worst = max(worst, e)
    print(f"float MUL_MAT C ABI vs f64: {len(cases)} layouts, worst NMSE {worst:.2e}")
