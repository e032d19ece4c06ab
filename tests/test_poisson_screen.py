"""Screened Poisson (poisson.py's point_weight) on the CPU: the float64 restatement of the rule
(oracle/poisson_screen_oracle.py) against the moments taken directly from the points, the
Galerkin identity P^T S_f P = S_c, a direct sparse solve, and the unscreened oracle at alpha = 0;
then the argument and command-line refusals, none of which touches the GPU."""
import math

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import poisson
from oracle import poisson_oracle as O
from oracle import poisson_screen_oracle as Q


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("depth", [6, 7])
def test_coarsened_moments_equal_moments_from_the_points(depth):
    p, _ = O.sphere(30_000, seed=3, noise=0.01)
    g = O.grid(p, depth)
    levels = Q.level_moments(p, g)
    assert len(levels) == depth - 2                             # N .. 8 nodes per axis
    for l, (keys, M) in enumerate(levels):
        dk, dM = Q.moments(p, g, l)
        assert np.array_equal(keys, dk)
        assert _rel(M, dM) <= 1e-12, l
        assert np.allclose(M[:, 0].sum(), len(p))               # every point lands in one cell


def test_galerkin_identity_of_the_screening_matrix():
    """P^T S_f P = S_c for random points whose cells keep clear of the outer layer and of the
    unstored coarse node n: trilinear prolongation reproduces a coarse trilinear function."""
    rng = np.random.default_rng(11)
    nf, nc = 32, 16
    h = 0.5
    g = dict(h=h, N=nf, lo=np.zeros(3, np.int64), centre=np.zeros(3))
    p = rng.uniform(2.0 * h, (nf - 3.0) * h, (5000, 3)).astype(np.float32)
    kf, Mf = Q.moments(p, g, 0)
    kc, Mc = Q.coarsen(kf, Mf, nf)
    Sf, _ = Q.screen_matrix(kf, Mf, nf, nf)
    Sc, _ = Q.screen_matrix(kc, Mc, nc, nc + 1)
    P = Q.prolongation(nc)
    G = (P.T @ Sf @ P).toarray()
    assert _rel(G, Sc.toarray()) <= 1e-12


def _system(depth, alpha=4.0):
    p, n = O.sphere(4000, seed=1)
    N = 1 << depth
    h = float(np.float32(1.1 * 2 / N))
    g = dict(h=h, N=N, lo=np.full(3, -N // 2, np.int64), centre=np.zeros(3))
    V, _, _ = O.splat(p, n, np.full((len(p), 3), 255.0), g)
    b = O.divergence(V, h)
    chi0, _, _ = O.multigrid(b, h)
    t = O.iso_level(chi0, p, g)
    return Q.screened_system(p, g, b, t, alpha), chi0, h


# depth 5 only: at depth 6 SuperLU's fill-in on the 27-point screened system over 62^3 unknowns
# takes longer than the rest of the CPU tier together (the run was stopped after 20 minutes)
@pytest.mark.parametrize("depth", [5])
def test_screened_multigrid_equals_the_direct_solve(depth):
    s, chi0, h = _system(depth)
    chi, cycles, ratios = Q.multigrid(s["b_s"], chi0, h, s["ops"], tol=1e-12, max_cycles=100)
    direct = Q.direct_solve(s["b_s"], h, s["S0"], s["g"])
    assert ratios[-1] <= 1e-12 and cycles <= 30
    assert np.abs(chi - direct).max() <= 1e-8 * np.abs(direct).max()
    # the default stopping rule converges well inside the cycle limit
    _, cycles, ratios = Q.multigrid(s["b_s"], chi0, h, s["ops"])
    assert ratios[-1] <= 1e-5 and cycles <= 10
    # screening moves the field: chi0 does not solve the screened system
    assert np.abs(direct - chi0).max() > 1e-3 * np.abs(direct).max()


def test_alpha_zero_reproduces_the_unscreened_oracle_exactly():
    p, n = O.sphere(20_000, seed=0, noise=0.002)
    want = O.poisson(p, normals=n, depth=6)
    got = Q.poisson(p, normals=n, depth=6, point_weight=0.0)
    assert got["screened_cycles"] == 0 and got["g"] == 0.0
    for k in ("chi", "keys", "tsdf", "weight", "color", "verts", "colours", "faces"):
        assert np.array_equal(got[k], want[k]), k
    assert got["iso"] == want["iso"]


def test_screened_sphere_and_cube_are_closed_and_the_cube_is_closer():
    p, n = O.sphere(20_000, seed=0, noise=0.002)
    r = Q.poisson(p, normals=n, depth=6, point_weight=4.0)
    d = np.abs(np.linalg.norm(r["verts"].astype(np.float64), axis=1) - 1.0)
    assert r["screened_ratios"][-1] <= 1e-5 and d.max() < r["grid"]["h"]
    assert O.mesh_oracle.is_closed_oriented(r["faces"])
    assert O.mesh_oracle.euler_characteristic(len(r["verts"]), r["faces"]) == 2
    p, n, q = Q.cube(60_000, seed=0)
    r0 = Q.poisson(p, normals=n, depth=6)
    r4 = Q.poisson(p, normals=n, depth=6, point_weight=4.0)
    d0, d4 = Q.cube_distance(r0["verts"], q), Q.cube_distance(r4["verts"], q)
    assert d4.mean() < d0.mean() and np.percentile(d4, 95) < np.percentile(d0, 95)
    assert O.mesh_oracle.signed_volume(r4["verts"], r4["faces"]) > 0


@pytest.mark.parametrize("bad", [-1.0, -1e-30, math.nan, math.inf, -math.inf, "4", True])
def test_poisson_mesh_refuses_a_bad_point_weight_before_using_the_gpu(bad):
    with pytest.raises(ValueError, match="point_weight must be"):
        poisson.poisson_mesh(torch.zeros(4, 3), normals=torch.zeros(4, 3), point_weight=bad)


def test_screening_is_counted_in_the_memory_check():
    n = 10_000
    assert poisson._bytes_needed(8, n, screen=True) > poisson._bytes_needed(8, n)
    assert poisson._bytes_needed(8, n, screen=True, n_cells=100) == \
        poisson._bytes_needed(8, n, screen=True) + 100 * poisson.SCREEN_BYTES_PER_CELL
    budget = poisson._bytes_needed(8, n, screen=True) - 1
    poisson._check_fits(8, n, budget)                          # fits unscreened
    with pytest.raises(Exception, match="with screening .*depth 7 would fit"):
        poisson._check_fits(8, n, budget, screen=True)


def test_cli_point_weight_flags(capsys, tmp_path):
    a, _ = poisson.parse_args(["--ply", "x", "--out", "y"])
    assert a.point_weight == 0.0
    a, _ = poisson.parse_args(["--ply", "x", "--out", "y", "--point_weight", "4"])
    assert a.point_weight == 4.0
    for bad in ("-1", "nan", "inf"):
        with pytest.raises(SystemExit):
            poisson.parse_args(["--ply", "x", "--out", "y", "--point_weight", bad])
        assert "--point_weight must be" in capsys.readouterr().err
    base = ["--root_dir", "x", "--scan", "scan1"]
    a = ep.parse_args(base + ["--mesh", "--mesh_method", "poisson", "--poisson_point_weight", "4"])
    assert a.poisson_point_weight == 4.0
    assert ep.parse_args(base + ["--mesh"]).poisson_point_weight is None
    for bad, msg in ((["--mesh", "--poisson_point_weight", "4"], "--poisson_point_weight needs"),
                     (["--poisson_point_weight", "4"], "--poisson_point_weight needs"),
                     (["--mesh", "--mesh_method", "tsdf", "--poisson_point_weight", "4"],
                      "--poisson_point_weight needs"),
                     (["--mesh", "--mesh_method", "poisson", "--poisson_point_weight", "-1"],
                      "finite number >= 0"),
                     (["--mesh", "--mesh_method", "poisson", "--poisson_point_weight", "nan"],
                      "finite number >= 0"),
                     (["--mesh", "--mesh_method", "poisson", "--poisson_point_weight", "inf"],
                      "finite number >= 0")):
        with pytest.raises(SystemExit):
            ep.parse_args(base + bad)
        assert msg in capsys.readouterr().err
