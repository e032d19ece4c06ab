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


# ------------------------------------------------------------------------------- oracle checks
# The inverse-mode checks of oracle/regress_fp64.py and oracle/inverse_depth_fp64.py against a
# float32 restatement of the kernels: the correct one passes, each injected defect fails where it
# was injected.
import test_feature_regress_fp64_oracle as FR                       # noqa: E402
from oracle import regress_fp64 as RG                                # noqa: E402

EPS_K3 = 2.0 ** -17              # the fp32 CUDA-core ceiling of the GPU checks
F32 = torch.float32


def _ladder_parts(B, h, w, D, kind, seed=0):
    """(first, step) of an inverse ladder over a wide range (near 0.5, far about 12): a float,
    per-item (B,) values or a per-pixel (B,h,w) first rung."""
    st = INV.steps_f32(torch.tensor([[0.5], [0.6]][:B]), torch.tensor([[0.24], [0.3]][:B]),
                       (8, 32, D), (1, 2, 4), B)
    un, s = st[0], st[2][2]
    if kind == "float":
        return float(un[0]), float(s[0])
    if kind == "batch":
        return torch.from_numpy(un), torch.from_numpy(s)
    g = np.random.default_rng(seed)
    cur = (0.6 + 9 * g.random((B, h // 2, w // 2))).astype(np.float32)
    return torch.from_numpy(INV.first_rung_f32(st, 2, D, cur)), torch.from_numpy(s)


def _ladder_defect(first, step, D, B, h, w, defect):
    fa, sa = INV._np32(first), INV._np32(step)
    if defect == "step_sign":
        sa = -sa
    elif defect == "step_of_item_0":
        sa = np.full(B, sa.reshape(-1)[0], dtype=np.float32)
    out = INV.ladder_f32(fa, sa, D + 1, B, h, w)
    return out[:, 1:] if defect == "plane_shift" else out[:, :D]


@pytest.mark.parametrize("kind", ["float", "batch", "map"])
def test_ladder_restatement_equals_materialize(kind):
    B, D, h, w = 2, 48, 6, 10
    first, step = _ladder_parts(B, h, w, D, kind)
    want = INV.ladder_f32(first, step, D, B, h, w)
    got = ops.Ladder(first, step, D, B, h, w, "cpu", inverse=True).materialize()
    assert np.array_equal(got.numpy(), want)
    # the coarse and fine stages of rules 3-4 are ladders
    st = INV.steps_f32(1.5, 0.38, (8, 32, 48), (1, 2, 4), B)
    assert np.array_equal(INV.ladder_f32(st[0], st[2][2], 48, B, h, w),
                          INV.hypotheses_f32(st, 2, 48, h, w))
    cur = np.random.default_rng(1).uniform(1.5, 80, (B, h // 2, w // 2)).astype(np.float32)
    assert np.array_equal(INV.ladder_f32(INV.first_rung_f32(st, 1, 32, cur), st[2][1], 32, B, h, w),
                          INV.hypotheses_f32(st, 1, 32, h, w, cur))


def _cascade16(terms, drop_tail=False):
    a0 = torch.zeros_like(terms[0])
    a1 = torch.zeros_like(a0)
    for i, t in enumerate(terms):
        a0 = a0 + t
        if i % 16 == 15:
            a1, a0 = a1 + a0, torch.zeros_like(a0)
    return a1 if drop_tail else a0 + a1


def regress_inv_f32(l, dv, input_is_prob=False, defect=None):
    """regress_inv_kernel in float32: depth = RN(1/ubar), ubar = sum p RN(1/dv) (Cascade16).
    defect 'uniform_avg': sum p dv, the uniform average; 'tail_dropped': the terms past the last
    full 16 (Cascade16's a0) are lost."""
    _, conf, idx, p = FR.regress_f32(l, dv, input_is_prob)
    D = l.shape[1]
    if defect == "uniform_avg":
        return _cascade16([p[:, d] * dv[:, d] for d in range(D)]), conf, idx, p
    v = 1.0 / dv
    ubar = _cascade16([p[:, d] * v[:, d] for d in range(D)], defect == "tail_dropped")
    return 1.0 / ubar, conf, idx, p


def regress_inv_bwd_f32(l, dv, gd):
    """regress_inv_bwd_kernel in float32."""
    e = FR._exp_f32(l - l.amax(1, keepdim=True))
    den = torch.zeros_like(gd)
    num = torch.zeros_like(gd)
    v = 1.0 / dv
    for d in range(l.shape[1]):
        den = den + e[:, d]
        num = (e[:, d].double() * v[:, d].double() + num.double()).to(F32)         # fmaf
    ubar = num / den
    depth = 1.0 / ubar
    g = -(depth * depth) * (gd / den)
    return e * (v - ubar.unsqueeze(1)) * g.unsqueeze(1)


def _k3_inv_inputs(seed, D, kind="map", B=2, h=10, w=14, scale=4.0):
    l = torch.randn(B, D, h, w, generator=torch.Generator().manual_seed(seed)) * scale
    first, step = _ladder_parts(B, h, w, D, kind, seed)
    return l, torch.from_numpy(INV.ladder_f32(first, step, D, B, h, w)), first, step


def _ok(rep, what):
    print(f"[oracle] {what}: {rep.describe()}")
    assert rep.ok, f"{what}: {rep.describe()}"


def _fails(rep, what):
    print(f"[oracle] defect {what}: {rep.describe()}")
    assert not rep.ok, f"defect {what} passed the bound: {rep.describe()}"
    return dict(zip(rep.names, rep.worst["at"]))


@pytest.mark.parametrize("is_prob", [False, True])
@pytest.mark.parametrize("D", [8, 24, 48, 56])
def test_regress_inverse_restatement_within_bound(D, is_prob):
    l, dv, _, _ = _k3_inv_inputs(30 + D, D, scale=30.0 if D == 8 else 4.0)
    if is_prob:
        l = torch.softmax(l, 1)
    depth, conf, idx, p = regress_inv_f32(l, dv, is_prob)
    reps = RG.check_regress(l, dv, depth, conf, idx, None if is_prob else p, is_prob, EPS_K3,
                            inverse=True)
    for k in ("prob", "depth", "conf"):
        if k in reps:
            _ok(reps[k], f"K3 inverse D={D} prob_in={is_prob} {k}")
    assert reps["index"][0] == 0, reps["index"]
    # the vector form takes the same bound
    vec = dv[0, :, 0, 0].contiguous()
    dvv = vec.view(1, D, 1, 1).expand_as(dv).contiguous()
    depth, conf, idx, p = regress_inv_f32(l, dvv, is_prob)
    _ok(RG.check_regress(l, vec, depth, conf, idx, None, is_prob, EPS_K3, inverse=True)["depth"],
        f"K3 inverse vector D={D}")


def test_regress_inverse_reference_matches_float64():
    """The inverse references equal INV.regress_f64 / regress_bwd_f64 applied to the planes
    whose reciprocals are exactly RN(1/dv), the values the kernels average."""
    l, dv, _, _ = _k3_inv_inputs(40, 32)
    v = RG.inverse_values(dv).double()
    ref = RG.regress_ref(l, dv, inverse=True)
    d64 = INV.regress_f64(l, 1.0 / v)[0]
    assert float(((1.0 / ref["depth"] - d64).abs() / d64).max()) < 1e-12
    gd = torch.randn(2, 10, 14, generator=torch.Generator().manual_seed(41))
    g64, _, A = RG.regress_bwd_ref(l, dv, gd, inverse=True)
    assert bool(((g64 - INV.regress_bwd_f64(l, 1.0 / v, gd)).abs() <= 1e-12 * A).all())


def test_regress_inverse_bwd_restatement_within_bound():
    for D in (8, 48):
        l, dv, _, _ = _k3_inv_inputs(50 + D, D)
        gd = torch.randn(2, 10, 14, generator=torch.Generator().manual_seed(D))
        g64, b0, A = RG.regress_bwd_ref(l, dv, gd, inverse=True)
        _ok(RG.check(regress_inv_bwd_f32(l, dv, gd), g64, b0, A, EPS_K3, ("b", "d", "y", "x")),
            f"K3 inverse backward D={D}")
        # the uniform backward of the same call is another gradient
        gu = FR.regress_bwd_f32(l, dv, gd)
        _fails(RG.check(gu, g64, b0, A, EPS_K3, ("b", "d", "y", "x")), f"uniform backward D={D}")


@pytest.mark.parametrize("D", [24, 40, 56])
@pytest.mark.parametrize("defect", ["uniform_avg", "tail_dropped"])
def test_defect_regress_inverse(defect, D):
    l, dv, _, _ = _k3_inv_inputs(60 + D, D)
    depth, conf, idx, p = regress_inv_f32(l, dv, defect=defect)
    _fails(RG.check_regress(l, dv, depth, conf, idx, p, False, EPS_K3, inverse=True)["depth"],
           f"K3 {defect} D={D}")


@pytest.mark.parametrize("defect", ["step_sign", "step_of_item_0", "plane_shift"])
def test_defect_ladder_inverse(defect):
    B, D, h, w = 2, 48, 10, 14
    l, dv, first, step = _k3_inv_inputs(70, D, "batch")
    bad = torch.from_numpy(_ladder_defect(first, step, D, B, h, w, defect))
    assert not torch.equal(bad, dv)
    at = _fails(RG.check_regress(l, dv, *regress_inv_f32(l, bad)[:3], eps=EPS_K3,
                                 inverse=True)["depth"], f"ladder {defect}")
    if defect == "step_of_item_0":
        assert at["b"] == 1
        assert torch.equal(bad[0], dv[0])


def first_rung_t32(st, level, D, cur, defect=None):
    """Rule 4 in torch float32, one rounding per operation.  defect 'no_clamp': the far clamp
    omitted; 'half_D_minus_1': (D-1)/2 steps instead of D/2."""
    un, uf, s = (torch.from_numpy(np.asarray(a)) for a in (st[0], st[1], st[2][level]))
    uc = 1.0 / torch.from_numpy(INV.upsample_f32(cur))
    sb = s.view(-1, 1, 1)
    half = torch.tensor((D - 1) * 0.5 if defect == "half_D_minus_1" else D * 0.5, dtype=F32)
    a = uc + half * sb
    if defect == "no_clamp":
        return a
    return torch.maximum(a, uf.view(-1, 1, 1) + torch.tensor(float(D - 1), dtype=F32) * sb)


@pytest.mark.parametrize("defect", [None, "no_clamp", "half_D_minus_1"])
def test_defect_first_rung(defect):
    """K4's first rung is checked bit for bit against first_rung_f32."""
    B, D = 2, 32
    st = INV.steps_f32(torch.tensor([[1.5], [0.9]]), torch.tensor([[0.38], [0.61]]), (8, D, 48),
                       (1, 2, 4), B)
    cur = np.random.default_rng(2).uniform(1.6, 6, (B, 6, 9)).astype(np.float32)
    cur[:, :2, :3] = 500.0                                   # beyond the far plane: clamped
    want = INV.first_rung_f32(st, 1, D, cur)
    clamp = INV.first_rung_f32(st, 1, D, np.full((B, 1, 1), 500.0, np.float32))
    clamped = want == clamp[:, :1, :1]
    assert clamped[:, :4, :6].all() and clamped.mean() < 0.5
    got = first_rung_t32(st, 1, D, cur, defect).numpy()
    if defect is None:
        assert np.array_equal(got, want)
        return
    diff = got != want
    print(f"[oracle] defect K4 {defect}: {int(diff.sum())} differing pixels, first at "
          f"{tuple(np.argwhere(diff)[0])}")
    if defect == "no_clamp":            # exactly the clamped pixels
        assert np.array_equal(diff, clamped)
    else:                               # every pixel the clamp leaves alone
        assert diff[~clamped].all()
