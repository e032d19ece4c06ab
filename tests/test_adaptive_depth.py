"""Adaptive depth ranges (README "Adaptive depth ranges", rule in csrc/regress.cu) without a GPU:
the float32 restatement of the planes against float64, the floor / clamp / NaN cases, the
refusals, the lambda constants, Ladder.materialize() with a step map, the spread bound against a
float32 evaluation, and the model and command-line switches."""
import os
import re

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, ops
from oracle import adaptive_depth_fp64 as AD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
ULP = 2.0 ** -24


def _inputs(B, hi, wi, seed, dmin=425.0, spread_scale=8.0):
    g = torch.Generator().manual_seed(seed)
    cur = dmin + 500.0 * torch.rand(B, hi, wi, generator=g)
    spread = spread_scale * torch.rand(B, hi, wi, generator=g)
    return cur, spread


@pytest.mark.parametrize("D", [2, 8, 32])
@pytest.mark.parametrize("step", [2.5, "per_item"])
def test_restatement_against_float64(D, step):
    cur, spread = _inputs(2, 6, 10, D)
    g = torch.tensor([[2.5], [5.3]]) if step == "per_item" else step
    h32 = AD.hypotheses_f32(cur, spread, D, g).astype(np.float64)
    h64 = AD.hypotheses_f64(cur, spread, D, g)
    lo, st = AD.window_f32(cur, spread, D, g)
    # r, lo, hi, hi - lo, the division, the product and the sum each round once
    k = np.arange(D).reshape(1, -1, 1, 1)
    bound = 8 * ULP * (np.abs(h64) + np.abs(lo)[:, None] + (np.abs(st) * (D - 1))[:, None] * 2) \
        + 4 * ULP * np.abs(st)[:, None] * k
    assert np.all(np.abs(h32 - h64) <= bound)
    # the planes are increasing and span [lo, ~hi]
    assert np.all(np.diff(h32, axis=1) > 0)


def test_floor_clamp_and_nan():
    B, hi, wi, D = 1, 2, 2, 8
    # constant maps upsample to the same constant
    cur = torch.full((B, hi, wi), 100.0)
    spread = torch.zeros(B, hi, wi)
    lo, st = AD.window_f32(cur, spread, D, 2.0)
    assert np.all(lo == f32(98.0)) and np.all(st == f32(f32(4.0) / f32(7)))   # floor: r = g
    spread = torch.full((B, hi, wi), 10.0)
    lo, st = AD.window_f32(cur, spread, D, 2.0)
    assert np.all(lo == f32(85.0)) and np.all(st == f32(f32(30.0) / f32(7)))  # r = 1.5 s
    cur = torch.full((B, hi, wi), 1.0)
    lo, st = AD.window_f32(cur, spread, D, 2.0)
    assert np.all(lo == f32(1e-7))                                            # clamp
    assert np.all(st == f32((f32(16.0) - f32(1e-7)) / f32(7)))
    spread = torch.full((B, hi, wi), float("nan"))
    cur = torch.full((B, hi, wi), 100.0)
    lo, st = AD.window_f32(cur, spread, D, 2.0)
    assert np.all(lo == f32(98.0))                                            # NaN spread: r = g
    cur = torch.full((B, hi, wi), float("nan"))
    lo, st = AD.window_f32(cur, torch.zeros(B, hi, wi), D, 2.0)
    assert np.all(lo == f32(1e-7)) and np.all(np.isnan(st))                   # NaN c propagates
    assert np.all(np.isnan(AD.hypotheses_f32(cur, torch.zeros(B, hi, wi), D, 2.0)))


def test_refusals():
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    with pytest.raises(_lib.CasMVSError, match="at least 2 planes"):
        CascadeMVSNet(n_depths=[1, 32, 48], depth_sampling="adaptive")
    with pytest.raises(_lib.CasMVSError, match="at least 2 planes"):
        CascadeMVSNet(n_depths=[8, 1, 48], depth_sampling="adaptive")
    CascadeMVSNet(n_depths=[8, 32, 1], depth_sampling="adaptive")     # the coarsest is uniform
    m = CascadeMVSNet(depth_sampling="adaptive")
    m.n_depths = [1, 32, 48]
    with pytest.raises(_lib.CasMVSError, match="at least 2 planes"):
        m._adaptive()
    cur, spread = _inputs(1, 2, 2, 0)
    with pytest.raises(_lib.CasMVSError, match="D >= 2"):
        ops.adaptive_hypotheses(cur, spread, 1, 2.0)
    with pytest.raises(_lib.CasMVSError, match="per-pixel"):
        ops.Ladder(1.0, torch.ones(1, 4, 4), 8, 1, 4, 4, "cpu")
    with pytest.raises(_lib.CasMVSError, match="inverse"):
        ops.Ladder(torch.ones(1, 4, 4), torch.ones(1, 4, 4), 8, 1, 4, 4, "cpu", inverse=True)
    with pytest.raises(ValueError):
        CascadeMVSNet(depth_sampling="adaptive+inverse")


def test_lambda_constants_equal():
    src = open(os.path.join(ROOT, "casmvsnet_pl_b200", "csrc", "regress.cu")).read()
    m = re.search(r"constexpr float kAdaptiveLambda = ([0-9.]+)f;", src)
    assert m and float(m.group(1)) == ops.ADAPTIVE_LAMBDA == AD.LAMBDA


def test_ladder_materialize_equals_restatement():
    cur, spread = _inputs(2, 5, 7, 3)
    for D in (2, 8, 32):
        lo, st = AD.hypotheses_f32(cur, spread, D, torch.tensor([2.5, 5.3]), first_only=True)
        lad = ops.Ladder(torch.from_numpy(lo), torch.from_numpy(st), D, 2, 10, 14, "cpu")
        got = lad.materialize().numpy()
        assert got.shape == (2, D, 10, 14)
        assert np.array_equal(got.view(np.uint32), AD.ladder_f32(lo, st, D).view(np.uint32))
        full = AD.hypotheses_f32(cur, spread, D, torch.tensor([2.5, 5.3]))
        assert np.array_equal(got.view(np.uint32), full.view(np.uint32))


def _spread_f32(logits, hyp):
    """The kernel's spread in float32: softmax as regress_body forms it, dhat and the second pass
    in Cascade16 order."""
    lg = logits.numpy().astype(f32)
    dv = hyp.numpy().astype(f32)
    B, D, h, w = lg.shape
    m = lg.max(1, keepdims=True)
    e = np.exp((lg - m).astype(f32)).astype(f32)
    den = np.zeros((B, 1, h, w), f32)
    for d in range(D):
        den = (den + e[:, d:d + 1]).astype(f32)
    p = (e / den).astype(f32)

    def c16(terms):
        a0 = np.zeros((B, h, w), f32)
        a1 = np.zeros((B, h, w), f32)
        for d in range(D):
            a0 = (a0 + terms[:, d]).astype(f32)
            if (d + 1) % 16 == 0:
                a1 = (a1 + a0).astype(f32)
                a0[:] = 0
        return (a0 + a1).astype(f32)
    dhat = c16((p * dv).astype(f32))
    t = (dv - dhat[:, None]).astype(f32)
    return np.sqrt(c16((p * (t * t).astype(f32)).astype(f32))).astype(f32)


@pytest.mark.parametrize("D,scale", [(8, 1.0), (32, 4.0), (48, 30.0), (48, 1.0)])
def test_spread_float32_within_bound(D, scale):
    g = torch.Generator().manual_seed(D)
    logits = scale * torch.randn(2, D, 6, 9, generator=g)
    first = 425.0 + 400.0 * torch.rand(2, 1, 6, 9, generator=g)
    hyp = (first + 2.5 * torch.arange(D, dtype=torch.float32).view(1, -1, 1, 1)).contiguous()
    sig, bound = AD.spread_ref(logits, hyp)
    got = torch.from_numpy(_spread_f32(logits, hyp)).double()
    assert torch.all((got - sig).abs() <= bound)
    if scale == 30.0:
        # peaked probabilities: E[d^2] - dhat^2 in float32 cancels at these depths, and the bound
        # is tight enough to tell
        p = torch.softmax(logits, 1)
        dhat = (p * hyp).sum(1)
        naive = ((p * hyp * hyp).sum(1) - dhat * dhat).clamp_min(0).sqrt().double()
        assert not torch.all((naive - sig).abs() <= bound)


def test_model_switch_and_state_dict():
    from casmvsnet_pl_b200 import ABN
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    a = CascadeMVSNet(norm_act=ABN)
    b = CascadeMVSNet(norm_act=ABN, depth_sampling="adaptive")
    assert "adaptive" in CascadeMVSNet.DEPTH_SAMPLINGS
    assert a.depth_sampling == "uniform" and b.depth_sampling == "adaptive"
    assert a.state_dict().keys() == b.state_dict().keys()
    assert a.set_depth_sampling("adaptive").depth_sampling == "adaptive"
    assert a.set_depth_sampling("uniform").depth_sampling == "uniform"


def test_cli_flag_absent_unless_given():
    from casmvsnet_pl_b200 import eval_pipeline, train
    ap = train.build_parser()
    assert not hasattr(ap.parse_args([]), "depth_sampling")
    assert ap.parse_args(["--depth_sampling", "adaptive"]).depth_sampling == "adaptive"
    base = ["--dataset_name", "colmap", "--root_dir", "capture"]
    assert not hasattr(eval_pipeline.parse_args(base), "depth_sampling")
    assert eval_pipeline.parse_args(base + ["--depth_sampling", "adaptive"]).depth_sampling == "adaptive"
