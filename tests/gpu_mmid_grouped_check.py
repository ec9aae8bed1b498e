"""Run in a SUBPROCESS with GGML_B200_MMID_GROUPED=1: MUL_MAT_ID with the rows grouped per expert on the device and multiplied on the
tensor-core GEMM kernel (mmq_tc2.cu, GROUPED mode) against the CPU oracle; --time prints the device time of the Mixtral-like case (8 experts, 2 used,
512 tokens, 4096 x 4096 Q4_K) for the grouped path and for the per-pair mat-vec path.  Exit code 0 = all checks passed."""
import os
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import ggml_b200 as g  # noqa: E402
from oracle import oracle as O  # noqa: E402


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def invalid_ids_and_elements(orc, rng):
    """256 experts, 8 used, ids a strided view of wider rows, an expert with no tokens and one with more than a tile of them, and ids -1
    and n_expert, into a NaN-filled dst inside NaN-sentinel guard bands and a workspace of exactly the queried size (0xFF, then a guard band).  Rows
    of invalid ids must be exactly zero, as on the per-pair form; every other element within the fp16-route bound of oracle/mm.py; a
    second launch into zeros gives the same bits."""
    import ctypes as C
    from oracle import mm
    sentinel, guard = 0x7FC0DEAD, 4096
    t, ne, nu, M, K, ntok = O.Q4_K, 256, 8, 384, 1024, 96
    for nb1 in (1, nu):
        W = O.random_blocks(t, ne * M * K // 256, rng)
        X = rng.uniform(-1, 1, (ntok * nb1, K)).astype(np.float32)
        others = np.delete(np.arange(ne), [7, 200])
        wide = np.stack([rng.permutation(others)[:nu + 2] for _ in range(ntok)]).astype(np.int32)
        wide[:90, 0] = 7                                       # expert 7: 90 tokens (> 64, this launch's tile width); expert 200: none
        assert not (wide[:, :nu] == 200).any() and (wide[:, :nu] == 7).sum() == 90
        wide[3, 1], wide[40, 5], wide[41, 7], wide[95, 2] = -1, ne, -1, ne + 5
        ids = dev(wide)[:, :nu]
        a = g.MulMatIdArgs()
        a.type, a.K, a.M, a.n_expert, a.n_used, a.nb1cols, a.n_tok = t, K, M, ne, nu, nb1, ntok
        rb = g.row_size(t, K)
        a.nb01, a.nb02, a.nb11, a.nb12, a.ids_nb1 = rb, rb * M, K * 4, K * 4 * nb1, (nu + 2) * 4
        ws_size = int(g.lib().ggml_b200_mul_mat_id_workspace_size(C.byref(a)))
        buf = torch.full((ntok * nu * M + 2 * guard,), sentinel, dtype=torch.int32, device="cuda")
        y = buf[guard:guard + ntok * nu * M].view(torch.float32)
        wsb = torch.full((ws_size + guard,), 0xA5, dtype=torch.uint8, device="cuda")
        Wd, Xd = dev(W), dev(X)
        outs = []
        for fill, wfill in ((float("nan"), 0xFF), (0.0, 0x00)):
            y.fill_(fill); wsb[:ws_size].fill_(wfill)
            g.mul_mat_id(t, Wd, Xd, ids, M, K, ne, nu, nb1, ntok, out=y, workspace=wsb[:ws_size])
            torch.cuda.synchronize()
            assert bool((buf[:guard] == sentinel).all()) and bool((buf[guard + y.numel():] == sentinel).all()), "a write outside dst"
            assert bool((wsb[ws_size:] == 0xA5).all()), "a write past the workspace"
            outs.append(y.clone())
        Y = outs[0].view(ntok, nu, M)
        bad = (wide[:, :nu] < 0) | (wide[:, :nu] >= ne)
        yb = Y[torch.from_numpy(bad).cuda()]
        nz = int((yb != 0).sum())
        assert nz == 0, f"rows of invalid ids: {nz} of {yb.numel()} elements not zero ({int(torch.isnan(yb).sum())} NaN)"
        assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "not the same bits into a zero-filled dst and workspace"
        R = mm.Reference(orc, t, W, ne * M, K, device="cuda")
        Xr = X.reshape(ntok, nb1, K)
        worst = 0.0
        for tok in range(ntok):
            for e in range(nu):
                x = int(wide[tok, e])
                if 0 <= x < ne:
                    r, bound = R(Xr[tok, e % nb1][None], "f16", rows=np.arange(x * M, (x + 1) * M))
                    worst = max(worst, float(mm.ratio(Y[tok, e][None], r, bound).max()))
        assert worst <= 1.0, worst
        print(f"ok grouped mul_mat_id q4_K 256x8 nb1cols={nb1}: {int(bad.sum())} invalid-id rows zero, worst |y - r| / bound {worst:.3g}", flush=True)


def main():
    assert os.environ.get("GGML_B200_MMID_GROUPED") == "1"
    g.lib()
    orc = O.Oracle()
    rng = np.random.default_rng(31)
    for (t, ne, nu, bc, ntok, M, K) in [(O.Q4_K, 8, 2, 0, 512, 1024, 1024), (O.Q8_0, 4, 1, 0, 100, 512, 512), (O.Q4_0, 8, 4, 1, 64, 300, 768), (O.Q6_K, 8, 2, 0, 129, 256, 2048),
                                        (O.Q4_K, 16, 4, 0, 37, 640, 256)]:
        nb1 = 1 if bc else nu
        W = O.random_blocks(t, ne * M * K // orc.blck_size(t), rng)
        X = rng.uniform(-1, 1, ntok * nb1 * K).astype(np.float32)
        # skewed routing: some experts get many tokens, some none
        p = rng.dirichlet(np.ones(ne) * 0.5)
        ids = np.stack([rng.choice(ne, size=nu, replace=False, p=p) for _ in range(ntok)]).astype(np.int32)
        Y = g.mul_mat_id(t, dev(W), dev(X), dev(ids), M, K, ne, nu, nb1, ntok).cpu().numpy()
        assert np.isfinite(Y).all()
        want = orc.mul_mat_id(t, W, X, ids, M, K, ne, nu, nb1, ntok)
        err = O.nmse(Y, want)
        assert err < 1e-4, (O.TYPE_NAMES[t], ne, nu, ntok, M, K, err)          # fp16 operands on the tensor-core path (reference gate 5e-4)
        print(f"ok grouped mul_mat_id {O.TYPE_NAMES[t]} experts={ne} used={nu} tokens={ntok} {M}x{K} nmse {err:.2e}", flush=True)
    invalid_ids_and_elements(orc, rng)
    if "--time" in sys.argv:
        t, ne, nu, ntok, M, K = O.Q4_K, 8, 2, 512, 4096, 4096
        W = dev(O.random_blocks(t, ne * M * K // 256, rng))
        X = dev(rng.uniform(-1, 1, ntok * nu * K).astype(np.float32))
        ids = dev(np.stack([rng.permutation(ne)[:nu] for _ in range(ntok)]).astype(np.int32))
        for _ in range(3):
            g.mul_mat_id(t, W, X, ids, M, K, ne, nu, nu, ntok)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            g.mul_mat_id(t, W, X, ids, M, K, ne, nu, nu, ntok)
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 100
        print(f"time grouped mul_mat_id q4_K 8x2 experts, 512 tokens, 4096x4096: {us:.1f} us = {2.0 * ntok * nu * M * K / us / 1e6:.0f} TFLOP/s", flush=True)
    print("grouped mul_mat_id OK")


if __name__ == "__main__":
    main()
