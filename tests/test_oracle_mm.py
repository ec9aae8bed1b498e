"""CPU-only: the f64 mat-mul reference of oracle/mm.py and its per-element bound against ggml-cpu's own MUL_MAT and MUL_MAT_ID
(oracle/_ref), for all 21 weight formats.  Every ggml-cpu element must lie within the integer-route bound of the reference, so that the
same bound on a device kernel means "no further from the exact value than ggml-cpu's own arithmetic allows".  The worst
|y - r| / bound per format must also stay above FLOOR: a bound loose enough to pass anything would fail that."""
import numpy as np
import pytest

from oracle import mm
from oracle import oracle as O

WEIGHT_TYPES = [t for t in sorted(O.TYPE_NAMES) if t not in (O.F32, O.F16, O.Q8_1, O.Q8_K)]
# worst ratio per format, measured on x86-64: 1.9e-3 (q5_K) to 3.6e-2 (q5_0); the floor is 4x under the smallest
FLOOR = 5e-4


def qk(t):
    return 32 if t in (O.Q4_0, O.Q4_1, O.Q5_0, O.Q5_1, O.Q8_0, O.IQ4_NL) else 256


def activations(rng, N, K):
    """uniform(-1, 1) rows, with a zero row and rows scaled by 2^-16 (fp16-subnormal Q8_0 scale), 2^-20 and 2^-30 (scale rounds to 0)"""
    X = rng.uniform(-1, 1, (N, K)).astype(np.float32)
    for i, s in zip(range(1, N), (0.0, 2.0 ** -16, 2.0 ** -20, 2.0 ** -30)):
        X[i] *= np.float32(s)
    return X


def shapes(t):
    """(M, N, K): one block, a K that is not a multiple of 256 for the 32-blocks, a long K; ragged M; n = 1..9"""
    Ks = [qk(t), 14336] + ([288, 4128] if qk(t) == 32 else [768])
    return [(7, 9, Ks[0]), (33, 5, Ks[1]), (5, 1, Ks[1])] + [(19, n, K) for n, K in zip((2, 3, 4, 6, 7, 8), Ks * 3)]


@pytest.mark.parametrize("t", WEIGHT_TYPES, ids=[O.TYPE_NAMES[t] for t in WEIGHT_TYPES])
def test_ggml_cpu_mul_mat_within_bound(t, ref, oracle):
    import torch
    rng = np.random.default_rng(100 + t)
    worst = 0.0
    for M, N, K in shapes(t):
        W = O.random_blocks(t, M * K // qk(t), rng)
        X = activations(rng, N, K)
        y, _ = ref.mul_mat(t, W, X, M, N, K, dev="CPU")
        r, bound = mm.Reference(oracle, t, W, M, K)(X, "int")
        q = mm.ratio(torch.from_numpy(y[0, 0]), r, bound)
        assert float(q.max()) <= 1.0, (M, N, K, float(q.max()), np.unravel_index(int(q.argmax()), q.shape))
        if N > 1:
            assert np.all(y[0, 0, 1] == 0)                                           # the zero row is exactly zero
        worst = max(worst, float(q.max()))
    print(f"{O.TYPE_NAMES[t]} worst {worst:.3e}")
    assert worst >= FLOOR, f"{O.TYPE_NAMES[t]}: worst |y - r| / bound {worst:.2e} < {FLOOR}: the bound is looser than it has to be"


@pytest.mark.parametrize("t", WEIGHT_TYPES, ids=[O.TYPE_NAMES[t] for t in WEIGHT_TYPES])
def test_ggml_cpu_mul_mat_id_within_bound(t, ref, oracle):
    import torch
    rng = np.random.default_rng(200 + t)
    ne, nu, ntok, M, K = 6, 2, 5, 17, 2 * qk(t) if qk(t) == 256 else 96
    for nb1 in (1, nu):
        W = O.random_blocks(t, ne * M * K // qk(t), rng)
        X = activations(rng, ntok * nb1, K)
        ids = np.stack([rng.permutation(ne)[:nu] for _ in range(ntok)]).astype(np.int32)
        y, _ = ref.mul_mat_id(t, W, X, ids, M, K, ne, nu, nb1, ntok, dev="CPU")
        R = mm.Reference(oracle, t, W, ne * M, K)
        Xr = X.reshape(ntok, nb1, K)
        for tok in range(ntok):
            for e in range(nu):
                rows = np.arange(ids[tok, e] * M, (ids[tok, e] + 1) * M)
                r, bound = R(Xr[tok, e % nb1][None], "int", rows=rows)
                q = mm.ratio(torch.from_numpy(y[tok, e][None]), r, bound)
                assert float(q.max()) <= 1.0, (nb1, tok, e, float(q.max()))
