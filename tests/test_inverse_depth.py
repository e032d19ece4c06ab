"""Inverse-depth plane sweep, host side: rules 1-2 (ops.inverse_steps) against the float32 /
float64 restatement of oracle/inverse_depth_fp64.py, the refusals of rule 1, the float32
restatement of the hypotheses against float64, and the switches of the model and the CLIs."""
import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, ops
from oracle import inverse_depth_fp64 as INV

RATIOS = [(1, 2, 4), (1, 2.5, 5.5)]
DEPTHS = [(8, 32, 48), (8, 8, 8), (32, 32, 32)]


def _steps_equal(got, want):
    un, uf, s = want
    assert np.array_equal(np.atleast_1d(np.asarray(got.u_near, np.float32)), un) or \
        float(got.u_near) == float(un[0])
    assert np.array_equal(np.broadcast_to(np.asarray(got.u_far, np.float32), uf.shape), uf)
    for g, w in zip(got.step, s):
        assert np.array_equal(np.broadcast_to(np.asarray(g, np.float32), w.shape), w)


@pytest.mark.parametrize("ratios", RATIOS)
@pytest.mark.parametrize("n_depths", DEPTHS)
def test_steps_float_and_cpu_tensor_match_restatement(n_depths, ratios):
    for dmin, dint, B in ((425.0, 2.65, 1), (1.5, 0.38, 1), (0.2, 1e-3, 1)):
        got = ops.inverse_steps(dmin, dint, n_depths, ratios, B)
        assert isinstance(got.u_near, float)
        _steps_equal(got, INV.steps_f32(dmin, dint, n_depths, ratios, B))
    dmin = torch.tensor([[425.0], [1.5]])
    dint = torch.tensor([[2.65], [0.38]])
    got = ops.inverse_steps(dmin, dint, n_depths, ratios, 2)
    assert got.u_near.shape == (2,) and got.u_near.device.type == "cpu"
    _steps_equal(got, INV.steps_f32(dmin, dint, n_depths, ratios, 2))


def test_steps_against_float64():
    """The float32 values are float64 rule 2 rounded once."""
    n_depths, ratios = (8, 32, 48), (1, 2, 4)
    un, uf, s = INV.steps_f32(1.5, 0.38, n_depths, ratios, 1)
    far = np.float32(np.float32(1.5) + np.float32(np.float32(0.38 * 4) * np.float32(47)))
    assert un[0] == np.float32(1 / 1.5) and uf[0] == np.float32(1 / np.float64(far))
    s_top = (1 / 1.5 - 1 / np.float64(far)) / 47
    assert s[2][0] == np.float32(s_top) and s[0][0] == np.float32(s_top * 1 / 4)


@pytest.mark.parametrize("dmin,dint", [(0.0, 2.65), (-1.0, 2.65), (425.0, 0.0), (425.0, -1.0),
                                       (float("nan"), 2.65), (425.0, float("inf")),
                                       (float("inf"), 2.65)])
def test_refusals_float(dmin, dint):
    with pytest.raises(_lib.CasMVSError, match="0 < near < far"):
        ops.inverse_steps(dmin, dint, [8, 32, 48], [1, 2, 4], 1)
    with pytest.raises(ValueError):
        INV.steps_f32(dmin, dint, [8, 32, 48], [1, 2, 4], 1)


def test_refusals_cpu_tensor_and_single_plane():
    with pytest.raises(_lib.CasMVSError, match="batch item 1"):
        ops.inverse_steps(torch.tensor([[425.0], [0.0]]), torch.tensor([[2.65], [2.65]]),
                          [8, 32, 48], [1, 2, 4], 2)
    with pytest.raises(_lib.CasMVSError, match="at least 2 planes"):
        ops.inverse_steps(425.0, 2.65, [8, 32, 1], [1, 2, 4], 1)


def test_hypotheses_restatement_against_float64():
    """The float32 restatement is within a few ulp of rules 3-4 in float64, increases with k and
    never passes the far plane by more than rounding."""
    g = np.random.default_rng(0)
    n_depths, ratios = (8, 32, 48), (1, 2, 4)
    st = INV.steps_f32(1.5, 0.38, n_depths, ratios, 2)
    far = 1 / st[1].astype(np.float64)
    coarse = INV.hypotheses_f32(st, 2, 48, 4, 5)
    assert (np.diff(coarse, axis=1) > 0).all()
    u64 = st[0].astype(np.float64)[:, None] - st[2][2].astype(np.float64)[:, None] * np.arange(48)
    # s*k and u_near - s*k are each rounded (at most half an ulp of u_near each), RN(1/u) adds
    # half an ulp of the depth: relative error <= eps*u_near/u_k + eps/2, eps = 2^-23
    eps = 2.0 ** -23
    bound = eps * st[0].astype(np.float64)[:, None] / u64 + eps / 2
    assert (np.abs(coarse[:, :, 0, 0] * u64 - 1) <= bound).all()
    cur = (1.5 + 73.5 * g.random((2, 6, 8))).astype(np.float32)
    cur[0, 0, 0] = 80.0                               # beyond far: the clamp holds
    fine = INV.hypotheses_f32(st, 1, 32, 12, 16, cur)
    assert (np.diff(fine, axis=1) > 0).all()
    assert (fine[:, -1] <= far[:, None, None] * (1 + 1e-6)).all()
    up = INV.upsample_f32(cur)
    ref = torch.nn.functional.interpolate(torch.from_numpy(cur).double()[:, None], scale_factor=2,
                                          mode="bilinear", align_corners=True)[:, 0].numpy()
    assert np.allclose(up, ref, rtol=1e-6, atol=0)


def test_model_switch_and_state_dict():
    from casmvsnet_pl_b200 import ABN
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    a = CascadeMVSNet(norm_act=ABN)
    b = CascadeMVSNet(norm_act=ABN, depth_sampling="inverse")
    assert a.depth_sampling == "uniform" and b.depth_sampling == "inverse"
    assert list(a.state_dict()) == list(b.state_dict())
    assert a.set_depth_sampling("inverse") is a and a.depth_sampling == "inverse"
    with pytest.raises(ValueError):
        a.set_depth_sampling("log")


def test_cli_flag_absent_unless_given():
    from casmvsnet_pl_b200 import eval_pipeline, train
    ap = train.build_parser()
    assert not hasattr(ap.parse_args([]), "depth_sampling")
    assert ap.parse_args(["--depth_sampling", "inverse"]).depth_sampling == "inverse"
    base = ["--dataset_name", "colmap", "--root_dir", "capture"]
    assert not hasattr(eval_pipeline.parse_args(base), "depth_sampling")
    assert eval_pipeline.parse_args(base + ["--depth_sampling", "inverse"]).depth_sampling == "inverse"


def test_inverse_hypotheses_refuses_a_cpu_device():
    st = ops.inverse_steps(1.5, 0.38, (8, 32, 48), (1, 2, 4), 1)
    with pytest.raises(_lib.CasMVSError, match="CUDA device"):
        ops.inverse_hypotheses(st, 2, 48, 8, 10, "cpu")


def test_tilted_capture_spans_a_wide_depth_range(tmp_path):
    from casmvsnet_pl_b200 import synth_scenes
    _, depths = synth_scenes.make_colmap(str(tmp_path / "c"), n_views=8, image_wh=(160, 128),
                                         n_points=500, seed=1, textured=True, tilt=2.25)
    for v, d in enumerate(depths):
        assert np.isfinite(d).all() and d.min() > 0 and d.max() / d.min() >= 9, v
    allv = np.concatenate([d.ravel() for d in depths])
    assert allv.max() / allv.min() >= 10
