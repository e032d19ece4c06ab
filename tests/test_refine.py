"""Mesh refinement on the CPU: the float64 oracle's rule (oracle/refine_oracle.py) recovers a known
offset of a planar mesh, constant-colour views move nothing, the tie rules and the tangent frame
hold, bad flags and arguments are refused, and the constants of refine.py, the oracle and
csrc/refine.cu agree."""
import os
import re

import numpy as np
import pytest

from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import refine
from oracle import refine_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_recovers_a_known_offset_of_a_planar_mesh():
    ims, Ps, srcs = O.plane_scene()
    v, f = O.grid_mesh(z=0.05)                               # 2.5 footprints above the plane
    out = O.refine_mesh(v, f, ims, Ps, srcs, 3)
    first = out["iterations"][0]
    rho = np.median(first["rho"][first["ref"] >= 0])
    assert 0.019 < rho < 0.021
    assert (first["ref"] >= 0).mean() > 0.8
    z = out["verts"][:, 2]
    assert np.median(np.abs(z)) < 0.05 * rho and np.sqrt(np.mean(z ** 2)) < 0.25 * rho
    assert np.abs(z).max() < 1.5 * rho
    # the exact plane stays put
    v0, _ = O.grid_mesh(z=0.0)
    z0 = O.refine_mesh(v0, f, ims, Ps, srcs, 3)["verts"][:, 2]
    assert np.sqrt(np.mean(z0 ** 2)) < 0.05 * rho


def test_constant_colour_views_move_nothing():
    ims, Ps, srcs = O.plane_scene(constant=(90, 140, 200))
    v, f = O.grid_mesh(z=0.05)
    out = O.refine_mesh(v, f, ims, Ps, srcs, 2)
    assert np.array_equal(out["verts"], v)
    assert all((it["conf"] == 0).all() and np.isnan(it["best"]).all() for it in out["iterations"])
    assert (out["iterations"][0]["ref"] >= 0).any()


def test_choice_ties_go_to_the_smaller_abs_k_then_the_smaller_k():
    nan = np.nan
    sk = np.full(2 * O.K + 1, nan)
    sk[O.K - 2], sk[O.K + 2] = 0.8, 0.8                      # k = -2 and +2 tie
    assert O.choose(sk)[:2] == (-2, 0.8)
    sk[O.K + 1] = 0.8                                        # +1 is nearer 0
    assert O.choose(sk)[0] == 1
    sk[O.K] = 0.8
    assert O.choose(sk)[0] == 0
    assert O.choose(np.full(2 * O.K + 1, nan))[0] == O.NO_K
    # a valid k = 0 stays unless k* beats it by MIN_GAIN
    sk = np.full(2 * O.K + 1, nan)
    sk[O.K], sk[O.K + 3] = 0.8, 0.8 + 0.5 * O.MIN_GAIN
    assert O.choose(sk) == (0, 0.8, 0.0)
    sk[O.K + 3] = 0.8 + 2 * O.MIN_GAIN
    assert O.choose(sk)[0] == 3
    # parabola: k* != 0 interior, both neighbours valid, negative curvature
    sk = np.full(2 * O.K + 1, nan)
    sk[O.K: O.K + 3] = [0.5, 0.9, 0.7]
    k, s, t = O.choose(sk)
    assert (k, s) == (1, 0.9) and t == pytest.approx((0.5 - 0.7) / (2 * (0.5 - 1.8 + 0.7)))
    sk[O.K] = nan                                            # a neighbour invalid: no sub-step
    assert O.choose(sk)[2] == 0.0
    sk = np.full(2 * O.K + 1, nan)
    sk[O.K - 1: O.K + 2] = [0.5, 0.9, 0.7]                   # k* = 0: no sub-step
    assert O.choose(sk) == (0, 0.9, 0.0)
    sk = np.full(2 * O.K + 1, nan)
    sk[-2:] = [0.4, 0.9]                                     # k* = K is not interior
    assert O.choose(sk)[:3] == (O.K, 0.9, 0.0)
    sk = np.full(2 * O.K + 1, 0.1)
    sk[O.K + 1: O.K + 4] = [0.25, 0.75, 0.75]                # k = 3 ties k* = 2: t = +0.5
    assert O.choose(sk)[:3] == (2, 0.75, 0.5)


def test_reference_ties_go_to_the_lower_view():
    x = np.zeros((1, 3), np.float32)
    n = np.array([[0.0, 0.0, 1.0]])
    eyes = [np.array([1.0, 0.0, 3.0]), np.array([-1.0, 0.0, 3.0]), np.array([0.0, 2.0, 3.0])]
    vis = np.array([[False, True, True]])
    ref, src = O.select(x, n, vis, eyes, [[1, 2], [2, 0], [0, 1]])
    assert ref[0] == 1 and list(src[0]) == [2, -1, -1, -1]   # view 0 is not visible
    vis[0, 0] = True
    ref, src = O.select(x, n, vis, eyes, [[2, 1], [2, 0], [0, 1]])
    assert ref[0] == 0 and list(src[0]) == [2, 1, -1, -1]    # views 0 and 1 tie: the lower
    ref, _ = O.select(x, n, np.array([[True, False, False]]), eyes, [[1, 2], [], []])
    assert ref[0] == -1                                      # no visible source: unseen


def test_tangent_frame_takes_the_axis_of_the_least_component():
    n = np.array([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [0.6, 0.0, 0.8], [0.48, 0.6, 0.64],
                  [0.6, 0.64, 0.48]])
    t1, t2 = O.frame(n)
    # ties to the lower axis: (0, 0, 1) and (0, 1, 0) take x, (0.6, 0, 0.8) takes y
    assert np.allclose(t1[0], [0, -1, 0]) and np.allclose(t1[1], [0, 0, 1])
    assert np.allclose(t1[2], np.cross([0, 1, 0], n[2]) / np.linalg.norm(np.cross([0, 1, 0], n[2])))
    assert np.allclose(t1[3], np.cross([1, 0, 0], n[3]) / np.linalg.norm(np.cross([1, 0, 0], n[3])))
    assert np.allclose(t1[4], np.cross([0, 0, 1], n[4]) / np.linalg.norm(np.cross([0, 0, 1], n[4])))
    for a, b, c in zip(n, t1, t2):
        assert np.allclose([a @ b, a @ c, b @ c], 0) and np.allclose(np.cross(a, b), c)


def test_constants_agree_with_the_kernels():
    src = open(os.path.join(ROOT, "casmvsnet_pl_b200", "csrc", "refine.cu")).read()
    kv = {m.group(1): float(m.group(2).rstrip("f")) for m in
          re.finditer(r"constexpr \w+ kRef(\w+) = ([-0-9.e]+f?);", src)}
    want = dict(R=refine.R, K=refine.K, Step=refine.STEP, SMax=refine.S_MAX,
                Spacing=refine.SPACING, MinGain=refine.MIN_GAIN,
                VarMin=refine.VAR_MIN, MinScore=refine.MIN_SCORE, Lambda=refine.LAMBDA,
                Pad=refine.PAD, MinCos=refine.MIN_COS, MaxBatch=refine.VIEW_BATCH,
                NoK=refine.NO_K)
    for name, value in want.items():
        assert kv[name] == value, name
    assert np.float32(kv["DepthScale"]) == np.float32(1 + refine.DEPTH_TOL)
    assert (O.SPACING, O.MIN_GAIN) == (refine.SPACING, refine.MIN_GAIN)
    assert (O.R, O.K, O.STEP, O.S_MAX, O.VAR_MIN, O.MIN_SCORE, O.LAMBDA, O.SMOOTH_ROUNDS, O.PAD,
            O.MIN_COS, O.NO_K) == (refine.R, refine.K, refine.STEP, refine.S_MAX, refine.VAR_MIN,
                                   refine.MIN_SCORE, refine.LAMBDA, refine.SMOOTH_ROUNDS,
                                   refine.PAD, refine.MIN_COS, refine.NO_K)
    assert O.DEPTH_SCALE == np.float32(1 + refine.DEPTH_TOL)


def test_bad_arguments_are_refused_before_the_gpu():
    with pytest.raises(ValueError, match="iterations"):
        refine.refine_mesh(None, None, None, [], [], [], iterations=0)
    with pytest.raises(ValueError, match="outside"):
        refine.check_sources([[1], [2]], 2)
    with pytest.raises(ValueError, match="source lists"):
        refine.check_sources([[1]], 2)
    assert refine.check_sources([[1], [0]], 2) == [[1], [0]]
    assert refine.pair_sources([(10, [12, 11, 99]), (12, [10])], [10, 11, 12]) == [[2, 1], [], [0]]


def test_flags_are_refused(capsys):
    base = ["--root_dir", "x"]
    for argv, msg in ((["--mesh_refine"], "--mesh_refine needs --mesh"),
                      (["--mesh", "--mesh_refine_iterations", "2"],
                       "--mesh_refine_iterations needs --mesh_refine"),
                      (["--mesh", "--mesh_refine", "--mesh_refine_iterations", "0"], ">= 1")):
        with pytest.raises(SystemExit):
            ep.parse_args(base + argv)
        assert msg in capsys.readouterr().err
    a = ep.parse_args(base + ["--mesh", "--mesh_refine"])
    assert ep._refine_iterations(a) == refine.ITERATIONS
    a = ep.parse_args(base + ["--mesh", "--mesh_refine", "--mesh_refine_iterations", "5"])
    assert ep._refine_iterations(a) == 5
    assert ep._refine_iterations(ep.parse_args(base + ["--mesh"])) is None
    with pytest.raises(SystemExit):
        refine.parse_args(["--ply", "a", "--cams", "b", "--images", "c", "--pair", "d", "--out",
                           "e", "--iterations", "0"])
