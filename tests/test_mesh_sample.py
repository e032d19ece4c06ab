"""Uniform surface sampling (mesh_sample.py) on its numpy restatement (oracle/mesh_sample_oracle.py):
counts, containment, coverage and the index decode; the error-cloud colour rule; the refusals and
the command-line errors of mesh scoring."""
import math

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import dtu_eval, mesh, mesh_sample, tnt_eval
from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200.fusion import write_ply
from oracle import mesh_sample_oracle as O


def _triangles(rng, n, scale=3.0):
    v = rng.uniform(-scale, scale, (3 * n, 3)).astype(np.float32)
    return v, np.arange(3 * n, dtype=np.int32).reshape(n, 3)


def test_counts_follow_the_longest_edge():
    rng = np.random.default_rng(0)
    v, f = _triangles(rng, 500)
    s = 0.37
    n, cnt = O.counts(v, f, s)
    for k, (a, b, c) in enumerate(v.astype(np.float64)[f]):
        L = max(math.dist(a, b), math.dist(b, c), math.dist(c, a))
        want = max(1, math.ceil(L / s))
        assert abs(n[k] - want) <= 1 and (n[k] == want or abs(L / s - round(L / s)) < 1e-9)
        assert cnt[k] == (n[k] + 1) * (n[k] + 2) // 2
    assert np.array_equal(O.offsets(cnt), np.concatenate([[0], np.cumsum(cnt)[:-1]]))
    # a point face and a huge face: n = 1 and the 2^16 clamp
    n, cnt = O.counts(np.float32([[0, 0, 0], [1e9, 0, 0], [0, 1e9, 0]]), [[0, 0, 0], [0, 1, 2]], 1.0)
    assert n.tolist() == [1, 65536] and cnt.tolist() == [3, 65537 * 65538 // 2]


def test_every_sample_lies_in_its_triangle():
    rng = np.random.default_rng(1)
    v, f = _triangles(rng, 200)
    pts, n, cnt, off = O.sample(v, f, 0.25)
    face = np.repeat(np.arange(len(f)), cnt)
    a, b, c = (v.astype(np.float64)[f[face, k]] for k in range(3))
    e1, e2, q = b - a, c - a, pts.astype(np.float64) - a
    # barycentric coordinates by least squares in the triangle's plane
    g = np.stack([np.einsum("ij,ij->i", e1, e1), np.einsum("ij,ij->i", e1, e2),
                  np.einsum("ij,ij->i", e2, e2)], 1)
    r = np.stack([np.einsum("ij,ij->i", q, e1), np.einsum("ij,ij->i", q, e2)], 1)
    det = g[:, 0] * g[:, 2] - g[:, 1] ** 2
    u = (g[:, 2] * r[:, 0] - g[:, 1] * r[:, 1]) / det
    w = (g[:, 0] * r[:, 1] - g[:, 1] * r[:, 0]) / det
    tol = 1e-5
    assert (u >= -tol).all() and (w >= -tol).all() and (u + w <= 1 + tol).all()
    resid = q - (u[:, None] * e1 + w[:, None] * e2)
    assert np.abs(resid).max() < 1e-5 * 6
    # the corners are samples: k = 0 is a, the last row's sample is b, the end of row 0 is c
    assert np.array_equal(pts[off], v[f[:, 0]])
    assert np.array_equal(pts[off + cnt - 1], v[f[:, 1]])
    assert np.array_equal(pts[off + n.astype(np.int64)], v[f[:, 2]])


def test_every_point_of_a_triangle_is_near_a_sample():
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(2)
    for trial in range(5):
        v, f = _triangles(rng, 1)
        s = float(rng.uniform(0.05, 0.3))
        pts = O.sample(v, f, s)[0]
        r1, r2 = rng.random(20000), rng.random(20000)
        flip = r1 + r2 > 1
        r1[flip], r2[flip] = 1 - r1[flip], 1 - r2[flip]
        a, b, c = v.astype(np.float64)
        q = a + r1[:, None] * (b - a) + r2[:, None] * (c - a)
        d, _ = cKDTree(pts.astype(np.float64)).query(q)
        eps = 4 * np.finfo(np.float32).eps * np.abs(v).max()
        assert d.max() <= s / math.sqrt(3) + eps, (trial, d.max(), s)


@pytest.mark.parametrize("n", [1, 2, 3, 7, 64, 999, 4000])
def test_decode_is_exact(n):
    i = np.concatenate([np.full(n + 1 - r, r) for r in range(n + 1)])
    j = np.concatenate([np.arange(n + 1 - r) for r in range(n + 1)])
    k = np.arange(len(i))
    assert len(k) == (n + 1) * (n + 2) // 2
    assert np.array_equal(O.row_start(i, n) + j, k)
    gi, gj = O.decode(k, np.full(len(k), n))
    assert np.array_equal(gi, i) and np.array_equal(gj, j)


def test_error_colours_follow_the_rule():
    d = np.array([0.0, 5.0, 10.0, 20.0, 2.5, 0.0, 10.0, 20.0, 2.5, 60.0])
    inside = np.array([True] * 5 + [False] * 5)
    want = [[255, 255, 255], [255, 128, 128], [255, 0, 0], [255, 0, 0], [255, 191, 191],
            [0, 0, 255], [0, 255, 0], [0, 255, 0], [0, 64, 191], [0, 255, 0]]
    got = dtu_eval.error_colours(d, inside)
    assert got.dtype == np.uint8 and got.tolist() == want


def _cpu_mesh():
    v = torch.tensor([[0, 0, 0], [1, 0, 0], [0, 1, 0]], dtype=torch.float32)
    return v, torch.tensor([[0, 1, 2]], dtype=torch.int32)


@pytest.mark.parametrize("spacing", [0, -0.1, math.nan, math.inf, True, "0.2", None])
def test_bad_spacing_is_refused(spacing):
    v, f = _cpu_mesh()
    with pytest.raises(ValueError, match="spacing"):
        mesh_sample.sample_surface(v, f, spacing)


def test_bad_meshes_are_refused():
    v, f = _cpu_mesh()
    with pytest.raises(ValueError, match="no faces"):
        mesh_sample.sample_surface(v, f[:0], 0.1)
    bad = v.clone()
    bad[1, 2] = math.nan
    with pytest.raises(ValueError, match="non-finite"):
        mesh_sample.sample_surface(bad, f, 0.1)
    with pytest.raises(ValueError, match="outside 0..2"):
        mesh_sample.sample_surface(v, f + 1, 0.1)
    with pytest.raises(ValueError, match="outside 0..2"):
        mesh_sample.sample_surface(v, f - 1, 0.1)
    with pytest.raises(ValueError, match="shape"):
        mesh_sample.sample_surface(v.double(), f, 0.1)
    with pytest.raises(ValueError, match="shape"):
        mesh_sample.sample_surface(v, f[:, :2], 0.1)
    with pytest.raises(ValueError, match="CUDA"):
        mesh_sample.sample_surface(v, f, 0.1)


def test_a_ply_without_faces_is_refused_naming_it(tmp_path):
    pts = tmp_path / "scan1.ply"
    write_ply(pts, np.zeros((4, 3), np.float32), np.zeros((4, 3), np.uint8))
    empty = tmp_path / "empty.ply"
    mesh.write_mesh_ply(empty, np.zeros((3, 3), np.float32), np.zeros((3, 3), np.uint8),
                        np.zeros((0, 3), np.int32))
    for p in (pts, empty):
        with pytest.raises(ValueError, match=str(p)):
            mesh_sample.load_mesh(str(p), "cuda:0")
    gt = tmp_path / "gt"
    gt.mkdir()
    with pytest.raises(ValueError, match="scan1.ply"):
        dtu_eval.main(["--mesh_dir", str(tmp_path), "--gt_dir", str(gt), "--scans", "1"])
    with pytest.raises(TypeError):
        mesh_sample.load_mesh(np.zeros((3, 3)), "cuda:0")


def test_command_line_errors(tmp_path):
    with pytest.raises(SystemExit):
        dtu_eval.main(["--gt_dir", str(tmp_path)])                      # neither source
    with pytest.raises(SystemExit):
        dtu_eval.main(["--ply_dir", "a", "--mesh_dir", "b", "--gt_dir", str(tmp_path)])
    common = ["--run_dir", "r", "--gt_dir", "g", "--scene", "Barn"]
    with pytest.raises(SystemExit):
        tnt_eval.main(common)                                           # neither source
    with pytest.raises(SystemExit):
        tnt_eval.main(common + ["--ply", "a.ply", "--mesh", "b.ply"])
    base = ["--root_dir", "x", "--scan", "scan1"]
    with pytest.raises(SystemExit):
        ep.parse_args(base + ["--mesh_score", "--dtu_gt", "gt"])        # no --mesh
    with pytest.raises(SystemExit):
        ep.parse_args(base + ["--mesh", "--mesh_score"])                # no ground truth
    a = ep.parse_args(base + ["--mesh", "--mesh_score", "--dtu_gt", "gt"])
    assert a.mesh_score and not ep.parse_args(base + ["--mesh"]).mesh_score


def test_run_scan_refuses_mesh_score_without_a_mesh_or_ground_truth():
    with pytest.raises(ValueError, match="mesh_score"):
        ep.run_scan(None, None, mesh_score=True, dtu_gt="gt")
    with pytest.raises(ValueError, match="mesh_score"):
        ep.run_scan(None, None, mesh_score=True, mesh_path="m.ply")
