"""CPU-only: the f64 references of oracle/attn.py against ggml-cpu (oracle/_ref/libggml_attn_probe.so), so that a wrong reference cannot
pass a wrong device kernel in tests/test_gpu_attention.py.
  - FLASH_ATTN_EXT within NMSE 5e-4 (the reference's own FA gate: ggml-cpu quantizes Q to K's vec-dot type and accumulates an f16 V in
    f16) on a grid that makes semantic mistakes large: ALiBi-style finite masks with -inf holes, max_bias 8 at 12 and 20 heads (both slope
    branches), softcap 30 over a wide score spread, GQA 32:8 and 32:1, permuted Q, K and V of different types, views of larger caches.
    ggml-cpu aborts on an f32 K, so f32 K / V are pinned against the f64 reference only (on the GPU);
  - SOFT_MAX within NMSE 1e-10: f16 and f32 masks with more rows than the input, ALiBi at 5 and 12 heads;
  - CPY into a view of a cache, bit-exact: Q8_0 as Oracle.quantize(simd_q8_0=True) (the AVX quantize_row_q8_0: ties to even), Q4_0 as
    Oracle.quantize (quantize_row_q4_0_ref), f16 as numpy's round-to-nearest-even; the cache outside the view untouched."""
from pathlib import Path

import numpy as np
import pytest

from oracle import attn as A
from oracle import oracle as O
from oracle.pool import F16, F32

FA_NMSE = 5e-4
SOFT_MAX_NMSE = 1e-10
G = Path(__file__).resolve().parent / "golden"


@pytest.fixture(scope="module", autouse=True)
def need_probe():
    if not (O.REF_DIR / "libggml_attn_probe.so").exists():
        pytest.skip("libggml_attn_probe.so not built (oracle/_ref needs the reference tree)")


FA_CPU_CASES = [
    A.FaCase(64, 37, 5, 32, 8, O.Q8_0, O.Q8_0, mask="finite", seed=1),
    A.FaCase(128, 70, 3, 32, 1, O.F16, O.F16, mask="causal", permute_q=True, seed=2),
    A.FaCase(64, 50, 4, 12, 12, O.F16, O.F16, mask="finite", max_bias=8.0, seed=3),
    A.FaCase(64, 50, 4, 20, 4, O.Q4_0, O.Q4_0, mask="finite", max_bias=8.0, seed=4),
    A.FaCase(64, 33, 2, 8, 8, O.F16, O.F16, mask="causal", softcap=30.0, seed=5),
    A.FaCase(256, 19, 3, 4, 2, O.Q4_K, O.Q6_K, mask="finite", ne3=2, seed=6),
    A.FaCase(64, 29, 7, 4, 4, O.F16, O.Q8_0, mask="causal", seed=7),
    A.FaCase(256, 9, 1, 4, 1, O.IQ2_XXS, O.IQ4_XS, mask="finite", seed=8),
    A.FaCase(40, 5, 1, 2, 2, O.F16, O.F16, seed=9),
]


@pytest.mark.parametrize("case", FA_CPU_CASES, ids=str)
def test_flash_attn_reference_matches_ggml_cpu(case):
    d = A.fa_data(case)
    ref = A.flash_attn_reference(case, d)
    cpu = A.flash_attn_ext("CPU", case, d)
    e = O.nmse(cpu, ref)
    # a reference that ignored the mask, the slopes, the softcap or the head mapping would be off by far more than the gate
    assert e <= FA_NMSE, (str(case), e)
    print(f"{case}: ggml-cpu vs f64 NMSE {e:.2e}")


def test_flash_attn_reference_semantics_are_visible():
    """the grid's masks, slopes and softcap each move the result far beyond the gate: a reference that dropped one of them would fail"""
    for case in (FA_CPU_CASES[0], FA_CPU_CASES[3], FA_CPU_CASES[4]):
        d = A.fa_data(case)
        cpu = A.flash_attn_ext("CPU", case, d)
        wrong = [(case, A.FaData(**{**d.__dict__, "mask": None}))]
        if case.max_bias:
            wrong.append((A.FaCase(**{**case.__dict__, "max_bias": 0.0}), d))
        if case.softcap:
            wrong.append((A.FaCase(**{**case.__dict__, "softcap": 0.0}), d))
        for c, dd in wrong:
            assert O.nmse(cpu, A.flash_attn_reference(c, dd)) > 100 * FA_NMSE, str(c)


SOFT_MAX_CPU_CASES = [
    A.SoftMaxCase((33, 4, 5, 1), F16, 8, scale=0.5, max_bias=8.0, seed=1),
    A.SoftMaxCase((129, 3, 12, 2), F32, 4, scale=0.125, max_bias=8.0, seed=2),
    A.SoftMaxCase((1025, 2, 3, 1), F16, 64, scale=1.0, seed=3),
    A.SoftMaxCase((32, 5, 1, 1), scale=2.0, seed=4),
]


@pytest.mark.parametrize("case", SOFT_MAX_CPU_CASES, ids=str)
def test_soft_max_reference_matches_ggml_cpu(case):
    x, mask = A.soft_max_data(case)
    e = O.nmse(A.soft_max("CPU", case, (x, mask)), A.soft_max_reference(case, x, mask))
    assert e <= SOFT_MAX_NMSE, (str(case), e)


def golden_x():
    return np.load(G / "act_q8.npz")["x"]


@pytest.mark.parametrize("case", A.cpy_grid(), ids=str)
def test_cpy_into_a_cache_is_what_the_oracle_restates(case):
    parent, cache = A.cpy_parent(case, golden_x()), A.cache_in(case)
    got = A.cpy("CPU", case, parent, cache)
    assert np.array_equal(got, A.cpy_expected(case, parent, cache)), str(case)


def test_q8_0_ties_separate_the_two_roundings():
    """on the tie inputs the _ref formula (roundf) and ggml-cpu's CPY (ties to even) differ: the Q8_0 bit-exact checks can tell them apart"""
    case = A.cpy_grid()[3]
    assert case.dst_type == O.Q8_0 and case.values == "ties"
    x = A.src_logical(case, A.cpy_parent(case))
    assert not np.array_equal(A.orc().quantize(O.Q8_0, x), A.orc().quantize(O.Q8_0, x, simd_q8_0=True))
