"""Dynamic consistency fusion without a GPU:

  * known answers of the rule (oracle/fusion_dynamic_fp64.level_of, geometric_mask) on hand-set
    errors: exactly k sources at level k pass, k - 1 fail, one tight source plus nine loose ones
    pass, errors just above a threshold move to the next level, S < 2 keeps nothing, and a zero
    or NaN reference depth is never consistent;
  * the rule's constants in fusion.py, the oracle and csrc/fusion.cu agree;
  * an fp32 restatement of geo_fuse_kernel<kDynamic> passes every float64 check on a scene and
    on the known-answer edge cases, and one with a defect fails;
  * eval_pipeline's --fusion flag: absent, today's namespace; dynamic with an explicit
    --min_geo_consistent, refused.
"""
import os
import re

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import eval_pipeline, fusion, synth_scenes
from oracle import fusion_dynamic_fp64 as FD
from oracle import fusion_fp64 as FF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _levels(*counts):
    """levels (S, 1) from (level, how many) pairs, in order."""
    return torch.tensor([lv for lv, n in counts for _ in range(n)], dtype=torch.int64).reshape(-1, 1)


# ------------------------------------------------------------------------------- the rule
@pytest.mark.parametrize("k", FD.LEVELS)
def test_k_sources_at_level_k(k):
    for S in range(k, 17):
        assert bool(FD.geometric_mask(_levels((k, k), (0, S - k)))), (k, S)
        # k - 1 sources at level k and none tighter: fails, whatever looser sources add below k
        assert not bool(FD.geometric_mask(_levels((k, k - 1), (0, S - k + 1)))), (k, S)
    if k < 10:
        # k - 1 at level k plus one at level k + 1: n_{k+1} = k < k + 1, fails
        assert not bool(FD.geometric_mask(_levels((k, k - 1), (k + 1, 1), (0, 2))))


def test_one_tight_and_nine_loose():
    assert bool(FD.geometric_mask(_levels((2, 1), (10, 9))))          # n_10 = 10, S = 10
    assert not bool(FD.geometric_mask(_levels((2, 1), (10, 8))))      # S = 9: n_9 = 1
    assert not bool(FD.geometric_mask(_levels((2, 1), (10, 8), (0, 7))))   # n_10 = 9
    assert bool(FD.geometric_mask(_levels((2, 1), (10, 9), (0, 6))))  # S = 16 counts to 10 only
    assert not bool(FD.geometric_mask(_levels((0, 16))))


def test_fewer_than_two_sources_keep_nothing():
    assert not bool(FD.geometric_mask(torch.zeros(0, 1, dtype=torch.int64)).any())
    for lv in (0, 2, 10):
        assert not bool(FD.geometric_mask(_levels((lv, 1))).any())
    assert bool(FD.geometric_mask(_levels((2, 2))))


@pytest.mark.parametrize("k", FD.LEVELS)
def test_threshold_edges(k):
    pix, dep = f32(k * k / 16), f32(k / 1300)
    nxt = k + 1 if k < 10 else 0
    below = lambda v: np.nextafter(v, f32(0))                          # noqa: E731
    above = lambda v: np.nextafter(v, f32(1e9))                        # noqa: E731
    assert int(FD.level_of(below(pix), 0.0)) == (k if k > 2 else 2)
    assert int(FD.level_of(below(pix), below(dep))) == k
    # on or just above a threshold: the next level
    assert int(FD.level_of(pix, below(dep))) == nxt
    assert int(FD.level_of(above(pix), below(dep))) == nxt
    assert int(FD.level_of(below(pix), dep)) == nxt
    assert int(FD.level_of(below(pix), above(dep))) == nxt
    assert FD.DEP_TH[k] == float(dep) and FD.PIX_TH[k] == float(pix)


def test_bad_reference_depths_are_never_consistent():
    rz = np.array([512, 0, -1, np.nan, np.inf], f32)
    for d in (f32(0), f32(-0.0), f32(np.nan)):
        with np.errstate(divide="ignore", invalid="ignore"):
            e_dep = np.abs((rz - d) / d)
        assert not np.isfinite(e_dep).any()
        assert (FD.level_of(np.zeros(5, f32), e_dep) == 0).all()
    # NaN pixel errors compare false too
    assert int(FD.level_of(f32(np.nan), 0.0)) == 0


def test_constants_agree_with_the_kernel():
    src = open(os.path.join(ROOT, "casmvsnet_pl_b200", "csrc", "fusion.cu")).read()
    c = {k: int(v) for k, v in re.findall(r"constexpr int (kDyn\w+) = (\d+);", src)}
    assert tuple(fusion.DYNAMIC_LEVELS) == tuple(range(c["kDynLevelMin"], c["kDynLevelMax"] + 1))
    assert fusion.DYNAMIC_PIX_DIV == c["kDynPixDiv"] and fusion.DYNAMIC_DEP_DIV == c["kDynDepDiv"]
    assert tuple(fusion.DYNAMIC_LEVELS) == FD.LEVELS
    assert (fusion.DYNAMIC_PIX_DIV, fusion.DYNAMIC_DEP_DIV) == (FD.PIX_DIV, FD.DEP_DIV)
    assert fusion.RULES == ("reference", "dynamic")


# ------------------------------------------------------------------------------- restatement
def restate(inp, defect=None):
    """geo_fuse_kernel<kDynamic> in torch float32 (CPU), one rounding per operation in the
    kernel's order, with an optional injected defect."""
    d = inp["depth_ref"].float()
    H, W = d.shape
    S = len(inp["depth_srcs"])
    y, x = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32),
                          indexing="ij")
    rs = np.asarray(inp["rs"], f32).reshape(-1, 12)
    sr = np.asarray(inp["sr"], f32).reshape(-1, 12)
    img_ref = inp["image_ref"].float()
    dsum, csum = d.clone(), img_ref.clone()
    levels = torch.zeros(S, H, W, dtype=torch.uint8)
    reproj = torch.zeros(S, H, W)
    t = lambda v: torch.tensor(float(v), dtype=torch.float32)          # noqa: E731

    def row(a, v):
        return ((t(a[0]) * v[0] + t(a[1]) * v[1]) + t(a[2]) * v[2]) + t(a[3])

    def sample(img, ix, iy, fx, fy):
        img3 = img if img.dim() == 3 else img.unsqueeze(-1)

        def tap(xx, yy):
            ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
            v = img3[yy.clamp(0, H - 1), xx.clamp(0, W - 1)]
            return torch.where(ok.unsqueeze(-1), v, torch.zeros_like(v))
        one = torch.tensor(1.0)
        w = [((one - fx) * (one - fy)), (fx * (one - fy)), ((one - fx) * fy), (fx * fy)]
        w = [v.unsqueeze(-1) for v in w]
        o = ((tap(ix, iy) * w[0] + tap(ix + 1, iy) * w[1]) + tap(ix, iy + 1) * w[2]) + tap(ix + 1, iy + 1) * w[3]
        return o if img.dim() == 3 else o[..., 0]

    for s in range(S):
        A, B = rs[s], sr[s]
        X, Y = x * d, y * d
        qx, qy, qz = row(A[0:4], (X, Y, d)), row(A[4:8], (X, Y, d)), row(A[8:12], (X, Y, d))
        xs, ys = qx / qz, qy / qz
        fin = torch.isfinite(xs) & torch.isfinite(ys)
        sx = torch.round((torch.where(fin, xs, 0.0) * 32).double()).clamp(-2.0 ** 31, 2.0 ** 31 - 1).long()
        sy = torch.round((torch.where(fin, ys, 0.0) * 32).double()).clamp(-2.0 ** 31, 2.0 ** 31 - 1).long()
        ix, iy = torch.div(sx, 32, rounding_mode="floor"), torch.div(sy, 32, rounding_mode="floor")
        fx, fy = (sx & 31).float() * (1 / 32), (sy & 31).float() * (1 / 32)
        ds = torch.where(fin, sample(inp["depth_srcs"][s].float(), ix, iy, fx, fy), torch.zeros_like(d))
        col = torch.where(fin.unsqueeze(-1), sample(inp["image_srcs"][s].float(), ix, iy, fx, fy),
                          torch.zeros(H, W, 3))
        U, V = xs * ds, ys * ds
        rx, ry, rz = row(B[0:4], (U, V, ds)), row(B[4:8], (U, V, ds)), row(B[8:12], (U, V, ds))
        dx, dy = rx / rz - x, ry / rz - y
        e_pix, e_dep = dx * dx + dy * dy, ((rz - d) / d).abs()
        lv = torch.zeros(H, W, dtype=torch.int64)
        for k in reversed(FD.LEVELS):
            th = t(k * k / 16) if defect != "pixel_not_squared" else t(k / 4)
            ok = (e_pix <= th) if defect == "le_threshold" else (e_pix < th)
            lv = torch.where(ok & (e_dep < t(k / 1300)), k, lv)
        m = lv > 0
        dsum = dsum + torch.where(m, rz, torch.zeros_like(rz))
        csum = csum + torch.where(m.unsqueeze(-1), col, torch.zeros_like(col))
        levels[s] = lv.to(torch.uint8)
        reproj[s] = torch.where(m, rz, torch.zeros_like(rz))
    lvl = levels.long()
    cnt = (lvl > 0).sum(0).int()
    keep = torch.zeros(H, W, dtype=torch.bool)
    for k in FD.LEVELS:
        if k <= S:
            counted = (lvl <= k) if defect == "count_level_zero" else ((lvl > 0) & (lvl <= k))
            keep |= counted.sum(0) >= k
    assert inp.get("proba_ref") is None, "the confidence test is fusion_fp64's, checked there"
    n1 = (cnt + 1).float()
    dref = dsum / n1
    image_refined = csum * (1 / n1).unsqueeze(-1)
    M = np.asarray(inp["ref2world"], f32).reshape(-1)
    Xr, Yr = x * dref, y * dref
    points = torch.stack([row(M[4 * r:4 * r + 4], (Xr, Yr, dref)) for r in range(3)], -1)
    return dict(level=levels, reproj=reproj, geo_count=cnt, mask_final=keep, depth_refined=dref,
                image_refined=image_refined, points=points)


@pytest.fixture(scope="module")
def scene10():
    views = synth_scenes.sphere_scene(11, (320, 256), seed=3, radius=150)
    inp = FF.scene_inputs(views, 10, seed=3, noise=0.002, proba=False)
    return inp


def test_restatement_passes(scene10):
    rep = FD.check_fuse_dynamic(scene10, restate(scene10))
    print(f"[fp64] dynamic restated S=10: {rep.describe()}")
    assert rep.ok, rep.describe()
    assert rep.ambiguous <= 2.0 ** -9 * rep.pairs, rep.describe()
    lv = restate(scene10)["level"].long()
    # the scene exercises the levels: several tight and loose levels occur, and the dynamic mask
    # differs from the fixed rule's
    hist = torch.bincount(lv.reshape(-1), minlength=11)
    assert (hist[2:11] > 0).sum() >= 8, hist


@pytest.mark.parametrize("name", [c[0] for c in FD.edge_cases() if c[0] != "confidence"])
def test_restatement_edge_cases(name):
    inp = dict(FD.edge_cases())[name]
    out = restate(inp)
    for exact in (True, False):
        rep = FD.check_fuse_dynamic(inp, out, exact)
        print(f"[fp64] dynamic restated {name}{' exact' if exact else ''}: {rep.describe()}")
        assert rep.ok, rep.describe()
    if name == "levels":
        # dx = 1/8, 3/8, 1/2, 5/8, 7/8, 1, 11/8, 9/4, 5/2, 3 px: levels on and between the thresholds
        assert out["level"][:, 5, 5].tolist() == [2, 2, 3, 3, 4, 5, 6, 10, 0, 0]


@pytest.mark.parametrize("defect", ["le_threshold", "pixel_not_squared", "count_level_zero"])
def test_injected_defect_fails(scene10, defect):
    cases = [("scene", scene10)] + [c for c in FD.edge_cases() if c[0] != "confidence"]
    caught = []
    for name, case in cases:
        bad = restate(case, defect)
        for exact in ((False,) if name == "scene" else (True, False)):
            rep = FD.check_fuse_dynamic(case, bad, exact=exact)
            if not rep.ok:
                caught.append((name, exact, rep.first_failure()))
    print(f"[fp64] dynamic defect {defect}: caught by {caught}")
    assert caught, f"{defect} passes every check"


# ------------------------------------------------------------------------------- eval_pipeline
def test_fusion_flag_is_opt_in():
    base = ["--root_dir", "r", "--scan", "scan1"]
    a = eval_pipeline.parse_args(base)
    assert not hasattr(a, "fusion") and a.min_geo_consistent == 5
    assert vars(eval_pipeline.parse_args(base + ["--fusion", "reference"])) == dict(vars(a), fusion="reference")
    assert eval_pipeline.parse_args(base + ["--fusion", "dynamic"]).fusion == "dynamic"
    assert eval_pipeline.parse_args(base + ["--fusion", "reference", "--min_geo_consistent", "3"]) \
        .min_geo_consistent == 3


@pytest.mark.parametrize("extra", [["--min_geo_consistent", "3"], ["--min_geo_consistent=5"]])
def test_dynamic_refuses_min_geo_consistent(capsys, extra):
    with pytest.raises(SystemExit) as e:
        eval_pipeline.parse_args(["--root_dir", "r", "--fusion", "dynamic"] + extra)
    assert e.value.code == 2
    assert "--min_geo_consistent" in capsys.readouterr().err


def test_rule_is_checked():
    with pytest.raises(ValueError, match="rule must be one of"):
        fusion.fuse_scan([], {}, {}, {}, {}, rule="fixed")
    with pytest.raises(SystemExit):
        eval_pipeline.parse_args(["--root_dir", "r", "--fusion", "fixed"])
