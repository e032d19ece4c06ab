"""Poisson surface reconstruction without a GPU: the float64 restatement (oracle/poisson_oracle.py)
against a direct sparse solve and against the geometry of analytic clouds, and the refusals of
the command line, the Python entry point and eval_pipeline's flags."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import poisson
from oracle import mesh_oracle as M
from oracle import poisson_oracle as O

CAMS = np.array([[3, 0, 0], [-3, 0, 0], [0, 3, 0], [0, -3, 0], [0, 0, 3], [0, 0, -3]], float)


@pytest.fixture(scope="module")
def sphere6():
    p, n = O.sphere(20_000, seed=0)
    return O.poisson(p, normals=n, depth=6)


def test_multigrid_equals_the_direct_solve_at_depth_5():
    p, n = O.sphere(3000, seed=1)
    N = 32
    h = float(np.float32(1.1 * 2 / N))
    g = dict(h=h, N=N, lo=np.full(3, -N // 2, np.int64), centre=np.zeros(3))
    V, _, _ = O.splat(p, n, np.full((len(p), 3), 255.0), g)
    b = O.divergence(V, h)
    chi, cycles, ratio = O.multigrid(b, h, tol=1e-12, max_cycles=100)
    direct = O.direct_solve(b, h)
    assert ratio <= 1e-12 and cycles <= 25
    assert np.abs(chi - direct).max() <= 1e-8 * np.abs(direct).max()
    # the default stopping rule converges well inside the cycle limit
    _, cycles, ratio = O.multigrid(b, h)
    assert ratio <= 1e-5 and cycles <= 10


def test_sphere_with_exact_normals_lies_within_one_node(sphere6):
    r = sphere6
    h = r["grid"]["h"]
    d = np.abs(np.linalg.norm(r["verts"].astype(np.float64), axis=1) - 1.0)
    assert len(r["faces"]) > 10_000 and r["dropped"] == 0
    assert d.max() < 1.0 * h
    # every level's boundary lies at the same place, so each V(2,2) cycle cuts the residual
    # several-fold: 1e-5 within 10 cycles, far from the 40-cycle cap
    assert r["ratio"] <= 1e-5 and r["cycles"] <= 10


def test_sphere_mesh_is_closed_with_outward_normals(sphere6):
    v, f = sphere6["verts"], sphere6["faces"]
    assert M.is_closed_oriented(f)
    assert M.euler_characteristic(len(v), f) == 2
    assert M.signed_volume(v, f) > 0
    # sign convention: f = chi - iso is negative inside, positive in free space
    g = sphere6["grid"]
    c = -g["lo"]                                             # the node at the origin
    assert sphere6["chi"][tuple(c)] - sphere6["iso"] < 0


def test_noisy_plane_gives_an_open_trimmed_mesh():
    p, n = O.plane(20_000, size=1.0, seed=0, noise=0.002)
    r = O.poisson(p, normals=n, depth=6)
    v, f, h = r["verts"], r["faces"], r["grid"]["h"]
    _, uc, _, _ = M.edge_counts(f)
    assert len(f) > 5000
    assert (uc == 1).any() and uc.max() <= 2                # open: it has a boundary
    # per axis, the mesh ends within 3 h of the samples' bounding box (the trim keeps nodes 2
    # nodes beyond the splat support, which reaches 1 node beyond a sample)
    lo, hi = p.min(0).astype(np.float64), p.max(0).astype(np.float64)
    assert (v >= lo - 3 * h).all() and (v <= hi + 3 * h).all()


def test_estimated_normals_are_accurate_and_face_the_cameras():
    p, _ = O.sphere(20_000, seed=2, noise=0.001)
    g = O.grid(p, 6)
    n, ok = O.estimate_normals(p, g, CAMS)
    assert ok.all()
    true = p.astype(np.float64) / np.linalg.norm(p.astype(np.float64), axis=1, keepdims=True)
    cos = (n * true).sum(1)
    assert np.degrees(np.arccos(np.clip(cos, -1, 1))).max() < 5.0
    near = CAMS[np.argmin(((p[:, None].astype(np.float64) - CAMS[None]) ** 2).sum(-1), axis=1)]
    assert ((n * (near - p)).sum(1) > 0).all()


def test_points_with_too_few_neighbours_or_a_line_get_no_normal():
    rng = np.random.default_rng(0)
    sph, _ = O.sphere(5000, seed=3)
    line = np.stack([np.linspace(3, 4, 200), np.zeros(200), np.zeros(200)], 1).astype(np.float32)
    lone = np.array([[-3.0, -3.0, -3.0], [-3.01, -3.0, -3.0]], np.float32)
    p = np.concatenate([sph, line, lone + rng.normal(0, 1e-4, lone.shape).astype(np.float32)])
    _, ok = O.estimate_normals(p, O.grid(p, 6), CAMS * 3)
    assert ok[:5000].all() and not ok[5000:].any()


def test_grid_rules():
    p, _ = O.sphere(1000)
    g = O.grid(p, 7)
    E = float((p.max(0).astype(np.float64) - p.min(0)).max())
    assert g["N"] == 128 and g["h"] == float(np.float32(1.1 * E / 128))
    cells = O.cell_index(p, g)
    assert cells.min() >= 0 and cells.max() < 128
    gp = poisson.grid(torch.from_numpy(p), 7)               # the product's grid, same rules
    assert gp["h"] == g["h"] and gp["lo"] == list(g["lo"]) and gp["N"] == 128


@pytest.mark.parametrize("pts, depth, match", [
    (np.zeros((5, 3)), 9, "zero extent"),
    (np.full((4, 3), np.nan), 9, "no finite point"),
    (np.eye(3), 5, "depth must be"),
    (np.eye(3), 11, "depth must be"),
])
def test_bad_clouds_and_depths_are_refused(pts, depth, match):
    t = torch.tensor(pts, dtype=torch.float32)
    with pytest.raises(ValueError, match=match):
        poisson.grid(t, depth)
    with pytest.raises(ValueError, match=match):
        O.grid(pts, depth)


def test_poisson_mesh_refuses_before_using_the_gpu():
    with pytest.raises(ValueError, match="depth must be"):
        poisson.poisson_mesh(torch.zeros(4, 3), normals=torch.zeros(4, 3), depth=11)
    with pytest.raises(ValueError, match="CUDA"):
        poisson.poisson_mesh(torch.zeros(4, 3), normals=torch.zeros(4, 3))


def _write_ply(path, xyz, normals=None, rgb=None):
    names = ["x", "y", "z"] + (["nx", "ny", "nz"] if normals is not None else [])
    dt = [(k, "<f4") for k in names] + ([(k, "u1") for k in ("red", "green", "blue")]
                                         if rgb is not None else [])
    v = np.empty(len(xyz), dtype=dt)
    v["x"], v["y"], v["z"] = xyz.T
    if normals is not None:
        v["nx"], v["ny"], v["nz"] = normals.T
    if rgb is not None:
        v["red"], v["green"], v["blue"] = rgb.T
    props = "".join(f"property {'float' if t == '<f4' else 'uchar'} {k}\n" for k, t in dt)
    with open(path, "wb") as f:
        f.write(f"ply\nformat binary_little_endian 1.0\nelement vertex {len(xyz)}\n{props}"
                "end_header\n".encode())
        v.tofile(f)


def test_cli_refuses_a_cloud_without_normals_or_cameras(tmp_path, capsys):
    p, _ = O.sphere(100)
    _write_ply(tmp_path / "c.ply", p)
    with pytest.raises(SystemExit):
        poisson.main(["--ply", str(tmp_path / "c.ply"), "--out", str(tmp_path / "m.ply")])
    err = capsys.readouterr().err
    assert "no normals" in err and "--cams" in err
    assert not (tmp_path / "m.ply").exists()
    with pytest.raises(SystemExit):
        poisson.main(["--ply", str(tmp_path / "c.ply"), "--out", str(tmp_path / "m.ply"),
                      "--depth", "12"])
    assert "--depth must be in 6..10" in capsys.readouterr().err


def test_cli_reads_ply_normals_colours_and_cameras(tmp_path):
    p, n = O.sphere(50)
    rgb = np.arange(150, dtype=np.uint8).reshape(50, 3)
    _write_ply(tmp_path / "n.ply", p, n, rgb)
    xyz, col, nrm = poisson.read_cloud(str(tmp_path / "n.ply"))
    assert np.array_equal(xyz, p) and np.array_equal(nrm, n) and np.array_equal(col, rgb)
    _write_ply(tmp_path / "plain.ply", p)
    xyz, col, nrm = poisson.read_cloud(str(tmp_path / "plain.ply"))
    assert col is None and nrm is None
    cams = poisson.camera_centres(os.path.join(os.path.dirname(__file__), "golden", "io"))
    from casmvsnet_pl_b200 import io as cio
    _, E, _ = cio.read_cam_file(os.path.join(os.path.dirname(__file__), "golden", "io",
                                             "00000000_cam.txt"))
    E = E.astype(np.float64)
    assert cams.shape == (4, 3)
    assert np.allclose(E[:3, :3] @ cams[0] + E[:3, 3], 0, atol=1e-6 * max(1, np.abs(E).max()))
    with pytest.raises(ValueError, match="no \\*_cam.txt"):
        poisson.camera_centres(str(tmp_path))


def test_eval_pipeline_mesh_method_flags(capsys):
    base = ["--root_dir", "x", "--scan", "scan1"]
    a = ep.parse_args(base + ["--mesh"])
    assert a.mesh_method == "tsdf" and a.poisson_depth is None
    a = ep.parse_args(base + ["--mesh", "--mesh_method", "poisson", "--poisson_depth", "8"])
    assert a.mesh_method == "poisson" and a.poisson_depth == 8
    for bad, msg in ((["--mesh_method", "poisson"], "needs --mesh"),
                     (["--mesh", "--mesh_method", "poisson", "--mesh_voxel", "0.5"], "--mesh_voxel"),
                     (["--mesh", "--poisson_depth", "8"], "--poisson_depth needs"),
                     (["--mesh", "--mesh_method", "tsdf", "--poisson_depth", "8"], "--poisson_depth needs"),
                     (["--mesh", "--mesh_method", "poisson", "--poisson_depth", "11"], "6..10")):
        with pytest.raises(SystemExit):
            ep.parse_args(base + bad)
        assert msg in capsys.readouterr().err
