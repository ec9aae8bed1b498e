"""CPU-only: the ctypes fronts of the one-node op probes (oracle/{attn,conv,core,grad,moe,pool,rope,sam,ssm,train,wkv}.py) against their libraries
(oracle/_ref/libggml_<family>_probe.so, over oracle/probe_harness.h).
  - each module's SIGNATURES names exactly the probe_* symbols its library exports, so a signature table cannot drift from the library;
  - every public probe function reports -1 for a device that does not exist ("NOPE"): with raw=True as its code, otherwise as a
    RuntimeError.  This is the harness's first exit path in all eleven libraries; no device is needed for it."""
import shutil
import subprocess

import numpy as np
import pytest

from oracle import attn as A
from oracle import conv as V
from oracle import core as K
from oracle import grad as G
from oracle import moe as M
from oracle import oracle as O
from oracle import pool as P
from oracle import rope as R
from oracle import sam as S
from oracle import ssm as SS
from oracle import train as TR
from oracle import wkv as W

MODULES = {"attn": A, "conv": V, "core": K, "grad": G, "moe": M, "pool": P, "rope": R, "sam": S, "ssm": SS, "train": TR, "wkv": W}


def need(family):
    so = O.REF_DIR / f"libggml_{family}_probe.so"
    if not so.exists():
        pytest.skip(f"{so.name} not built (oracle/_ref needs the reference tree)")
    return so


@pytest.mark.parametrize("family", sorted(MODULES))
def test_signatures_match_the_exported_probes(family):
    so = need(family)
    if shutil.which("nm") is None:
        pytest.skip("nm not installed")
    out = subprocess.run(["nm", "-D", "--defined-only", str(so)], check=True, capture_output=True, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if " T probe_" in line}
    assert set(MODULES[family].SIGNATURES) == exported


def _f32(*shape):
    return np.ones(shape, dtype=np.float32)


def _train_source():
    return P.Source(P.F32, (3, 2, 1, 1))


# (family, the probe_* symbol it reaches, a call on "NOPE" with a small valid input: its code, or "raises" for the functions without raw)
CALLS = [
    ("attn", "probe_flash_attn_ext", lambda: A.flash_attn_ext("NOPE", A.FaCase(32, 3, 1, 2, 1, O.F16, O.F16, mask="causal"), raw=True)),
    ("attn", "probe_soft_max", lambda: A.soft_max("NOPE", A.SoftMaxCase((8, 2, 3, 1), P.F16, 4, max_bias=8.0), raw=True)),
    ("attn", "probe_cpy", lambda: A.cpy("NOPE", A.CpyCase(P.Source(P.F32, (32, 2)), O.Q8_0, (32, 2), 4, 1), _f32(2, 32), np.zeros(136, np.uint8),
                                        raw=True)),
    ("core", "probe_get_rows", lambda: K.get_rows("NOPE", K.block_source(O.Q4_0, (32, 3)), np.zeros(54, np.uint8), np.zeros((1, 1, 2), np.int32),
                                                 raw=True)),
    ("core", "probe_binary", lambda: K.binary("NOPE", K.ADD, P.Source(P.F32, (4, 3)), _f32(3, 4), P.Source(P.F32, (4, 1)), _f32(1, 4), raw=True)),
    ("core", "probe_norm", lambda: K.norm("NOPE", True, 1e-6, P.Source(P.F32, (8, 2)), _f32(2, 8), raw=True)),
    ("core", "probe_unary", lambda: K.unary("NOPE", K.GELU_QUICK, _f32(5), raw=True)),
    ("core", "probe_scale_mask", lambda: K.scale_mask("NOPE", _f32(2, 3, 4), 0.5, 1, raw=True)),
    ("core", "probe_cpy", lambda: K.cpy("NOPE", 1, P.Source(P.F32, (4, 3), transpose=True), _f32(4, 3), raw=True)),
    ("core", "probe_norm_affine", lambda: K.norm_affine("NOPE", False, 1e-5, _f32(2, 8), _f32(8), _f32(8), raw=True)),
    ("core", "probe_scale_mask_softmax", lambda: K.scale_mask_softmax("NOPE", _f32(2, 3, 4), 0.5, 1, raw=True)),
    ("conv", "probe_im2col", lambda: V.im2col("NOPE", V.im2col_grid()[0], raw=True)),
    ("conv", "probe_mul_mat_f16", lambda: V.mul_mat_f16("NOPE", 4, 2, 8, raw=True)),
    ("conv", "probe_conv_1d", lambda: V.conv_1d("NOPE", 3, 2, 2, 8, 1, 0, 1, raw=True)),
    ("moe", "probe_argsort", lambda: M.argsort("NOPE", M.argsort_grid()[0], M.ASC, raw=True)),
    ("moe", "probe_sum_rows", lambda: M.sum_rows("NOPE", M.argsort_grid()[0])),
    ("pool", "probe_pool_2d", lambda: P.pool_2d("NOPE", P.pool_grid()[0], raw=True)),
    ("pool", "probe_upscale", lambda: P.upscale("NOPE", P.upscale_grid()[0], raw=True)),
    ("pool", "probe_leaky_relu", lambda: P.leaky_relu("NOPE", P.leaky_grid()[0], raw=True)),
    ("pool", "probe_repeat", lambda: P.repeat("NOPE", P.repeat_grid()[0], raw=True)),
    ("rope", "probe_rope", lambda: R.probe("NOPE", R.grid()[0])),
    ("sam", "probe_win_part", lambda: S.win_part("NOPE", S.win_part_grid()[0], raw=True)),
    ("sam", "probe_win_unpart", lambda: S.win_unpart("NOPE", S.win_unpart_grid()[0], raw=True)),
    ("sam", "probe_get_rel_pos", lambda: S.get_rel_pos("NOPE", S.rel_pos_grid()[0], raw=True)),
    ("sam", "probe_add_rel_pos", lambda: S.add_rel_pos("NOPE", S.add_rel_pos_grid()[0], raw=True)),
    ("sam", "probe_conv_transpose_2d", lambda: S.conv_transpose_2d("NOPE", S.conv_transpose_grid()[0], raw=True)),
    ("sam", "probe_sin_cos", lambda: S.sin_cos("NOPE", S.sin_cos_grid()[0], raw=True)),
    ("ssm", "probe_concat", lambda: SS.concat("NOPE", SS.concat_grid()[0], raw=True)),
    ("ssm", "probe_ssm_conv", lambda: SS.ssm_conv("NOPE", SS.conv_grid()[0], raw=True)),
    ("ssm", "probe_ssm_scan", lambda: SS.ssm_scan("NOPE", SS.scan_grid()[0], raw=True)),
    ("train", "probe_out_prod", lambda: TR.out_prod("NOPE", _train_source(), _train_source(), _f32(1, 1, 2, 3), _f32(1, 1, 2, 3), raw=True)),
    ("train", "probe_cross_entropy_loss", lambda: TR.cross_entropy_loss("NOPE", _f32(2, 3), _f32(2, 3), raw=True)),
    ("train", "probe_cross_entropy_loss_back", lambda: TR.cross_entropy_loss_back("NOPE", 1.0, _f32(2, 3), _f32(2, 3), raw=True)),
    ("train", "probe_opt_step_adamw", lambda: TR.opt_step_adamw("NOPE", _f32(4), _f32(4), _f32(4), _f32(4), _f32(7), raw=True)),
    ("train", "probe_argmax", lambda: TR.argmax("NOPE", _f32(2, 3), raw=True)),
    ("train", "probe_count_equal", lambda: TR.count_equal("NOPE", np.zeros(4, np.int32), np.zeros(4, np.int32), raw=True)),
    ("train", "probe_sum", lambda: TR.sum_("NOPE", _train_source(), _f32(1, 1, 2, 3), raw=True)),
    ("train", "probe_repeat_back", lambda: TR.repeat_back("NOPE", _train_source(), (3, 1), _f32(1, 1, 2, 3), raw=True)),
    ("train", "probe_step", lambda: TR.step("NOPE", _f32(4), raw=True)),
    ("grad", "probe_mul_mat_grad", lambda: G.mul_mat_grad("NOPE", G.GradCase(2, 1, 3), *G.GradCase(2, 1, 3).inputs(0), [0], [0], raw=True)),
    ("wkv", "probe_rwkv_wkv6", lambda: W.wkv("NOPE", W.grid(False)[0], raw=True)),
    ("wkv", "probe_gated_linear_attn", lambda: W.wkv("NOPE", W.grid(True)[0], raw=True)),
    ("wkv", "probe_sqr_sqrt", lambda: W.sqr_sqrt("NOPE", 0, _f32(4), raw=True)),
]
RAISES = {"probe_sum_rows", "probe_rope"}


def test_every_probe_is_called():
    assert {sym for _, sym, _ in CALLS} == {sym for m in MODULES.values() for sym in m.SIGNATURES}


def _call_ids():
    """each call's id: its symbol, prefixed by its family where an earlier family exports the same symbol (attn's and core's probe_cpy)"""
    ids = []
    for fam, sym, _ in CALLS:
        ids.append(f"{fam}-{sym}" if sym in ids else sym)
    return ids


@pytest.mark.parametrize("family, symbol, call", CALLS, ids=_call_ids())
def test_unknown_device_returns_minus_one(family, symbol, call):
    need(family)
    if symbol in RAISES:
        with pytest.raises(RuntimeError, match=r"returned -1$"):
            call()
    else:
        assert call() == -1


@pytest.mark.parametrize("gla", [False, True], ids=["wkv6", "gla"])
def test_wkv_token_override_reports_the_code(gla):
    """with T overridden (a T the case's result cannot be split by) raw=True still returns the probe's code"""
    need("wkv")
    assert W.wkv("NOPE", W.WkvCase(16, 2, 2, 2, gla=gla), raw=True, T=5) == -1
