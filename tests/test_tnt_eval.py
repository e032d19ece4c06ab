"""Tanks and Temples scoring without a GPU: readers and their refusals, Umeyama and the RANSAC
alignment, the restatement's crop, voxel means and nearest neighbours against brute force, the
synthetic scene's seeding and the command line's refusals."""
import json
import os

import numpy as np
import pytest

from casmvsnet_pl_b200 import synth_tnt
from casmvsnet_pl_b200 import tnt_eval as E
from oracle import tnt_eval_oracle as O


# ------------------------------------------------------------------------------ readers
def test_readers_round_trip(tmp_path):
    T = synth_tnt.similarity(np.random.default_rng(0))
    synth_tnt.write_trans(str(tmp_path / "t.txt"), T)
    assert np.array_equal(E.read_trans(str(tmp_path / "t.txt")), T)
    poses = [synth_tnt._rigid(synth_tnt.similarity(np.random.default_rng(k))) for k in range(4)]
    synth_tnt.write_log(str(tmp_path / "a.log"), poses)
    assert np.array_equal(E.read_log(str(tmp_path / "a.log")), np.stack(poses))
    assert np.array_equal(E.trajectory_from_log(str(tmp_path / "a.log")).centres,
                          np.stack(poses)[:, :3, 3])
    for axis in range(3):
        synth_tnt.write_crop(str(tmp_path / "c.json"), axis, -1, 2, [[1, 2, 3], [4, 5, 6], [7, 8, 0]])
        ax, lo, hi, poly = E.read_crop(str(tmp_path / "c.json"))
        assert (ax, lo, hi) == (axis, -1.0, 2.0)
        u, v = E.plane_axes(axis)
        assert np.array_equal(poly, np.array([[1, 2, 3], [4, 5, 6], [7, 8, 0]], float)[:, [u, v]])


@pytest.mark.parametrize("body, key", [
    ("1 0 0 0\n0 1 0 0\n0 0 1 0\n", "16"),
    ("1 0 0 0\n0 1 0 0\n0 0 1 0\n0 0 0 x\n", "not a number"),
    ("1 0 0 0\n0 1 0 0\n0 0 1 0\n0 0 1 1\n", "last row"),
])
def test_bad_trans_is_refused(tmp_path, body, key):
    p = tmp_path / "Barn_trans.txt"
    p.write_text(body)
    with pytest.raises(ValueError, match=key) as e:
        E.read_trans(str(p))
    assert "Barn_trans.txt" in str(e.value)


@pytest.mark.parametrize("body, key", [
    ("0 0 0\n1 0 0 0\n0 1 0 0\n0 0 1 0\n", "5 lines"),
    ("0 0\n1 0 0 0\n0 1 0 0\n0 0 1 0\n0 0 0 1\n", "3 integers"),
    ("0 0 0\n1 0 0 0\n0 1 0 0\n0 0 1 0\n0 0 0 nan\n", "finite"),
])
def test_bad_log_is_refused(tmp_path, body, key):
    p = tmp_path / "x.log"
    p.write_text(body)
    with pytest.raises(ValueError, match=key) as e:
        E.read_log(str(p))
    assert "x.log" in str(e.value)


@pytest.mark.parametrize("patch, key", [
    ({"orthogonal_axis": "W"}, "orthogonal_axis"),
    ({"axis_min": "a"}, "axis_min"),
    ({"axis_max": -5}, "axis_min must be <= axis_max"),
    ({"bounding_polygon": [[0, 0, 0]]}, "bounding_polygon"),
    ({"bounding_polygon": [[0, 0], [1, 1], [2, 0]]}, "bounding_polygon"),
])
def test_bad_crop_is_refused(tmp_path, patch, key):
    d = dict(orthogonal_axis="Z", axis_min=0, axis_max=1,
             bounding_polygon=[[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    d.update(patch)
    p = tmp_path / "Barn.json"
    p.write_text(json.dumps(d))
    with pytest.raises(ValueError, match=key) as e:
        E.read_crop(str(p))
    assert "Barn.json" in str(e.value)
    p.write_text("{not json")
    with pytest.raises(ValueError, match="not a JSON"):
        E.read_crop(str(p))


# ------------------------------------------------------------------------------ alignment
@pytest.mark.parametrize("reflect", [False, True])
def test_umeyama_recovers_a_similarity(reflect):
    rng = np.random.default_rng(1)
    T = synth_tnt.similarity(rng)
    s = rng.normal(size=(50, 3))
    if reflect:   # nearly planar points, where a reflection fits almost as well as the rotation
        s[:, 2] *= 1e-3
    d = s @ T[:3, :3].T + T[:3, 3]
    for fn in (E.umeyama, O.umeyama):
        got = fn(s, d)
        assert np.abs(got - T).max() < 1e-9
        assert np.linalg.det(got[:3, :3]) > 0


def test_ransac_recovers_T0_with_outliers_and_missing_cameras(tmp_path):
    rng = np.random.default_rng(2)
    T = synth_tnt.similarity(rng)
    gt = rng.uniform(-5, 5, (60, 3))
    keep = np.sort(rng.choice(60, 50, replace=False))          # 10 cameras missing
    rec = (gt[keep] - T[:3, 3]) @ np.linalg.inv(T[:3, :3]).T
    bad = rng.choice(50, 10, replace=False)                      # 20 % outliers
    rec[bad] += rng.normal(size=(10, 3)) * 3
    names = [f"{k:04d}.png" for k in range(60)]
    (tmp_path / "images").mkdir()
    for n in names:
        (tmp_path / "images" / n).write_bytes(b"")
    traj = E.Trajectory(rec, [names[k] for k in keep])
    T0, al = E.align(traj, gt, np.eye(4), str(tmp_path / "images"), seed=0)
    assert al == dict(pairs=50, inliers=40)
    assert np.abs(T0 - T).max() < 1e-9
    T1, _ = E.align(traj, gt, np.eye(4), str(tmp_path / "images"), seed=0)
    assert np.array_equal(T0, T1)
    with pytest.raises(ValueError, match="--images"):
        E.pair_cameras(traj, 60)
    with pytest.raises(ValueError, match="at least 6"):
        E.ransac_align(rec[:5], gt[:5])


# ------------------------------------------------------------------------------ restatement
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_oracle_crop_on_vertices_edges_and_bounds(axis):
    poly = np.array([[0.0, 0.0], [4.0, 0.0], [4.0, 2.0], [0.0, 2.0]])
    u, v = O.plane_axes(axis)

    def pt(pu, pv, pa=0.5):
        p = np.zeros(3, np.float32)
        p[u], p[v], p[axis] = pu, pv, pa
        return p

    cases = [  # (point, inside) under CropInPolygon's half-open rule
        (pt(2, 1), True), (pt(5, 1), False),
        (pt(0, 1), False),      # left edge: u must exceed the lower vertex u
        (pt(4, 1), True),       # right edge: u <= the upper vertex u
        (pt(2, 0), False),      # bottom edge: the node equals p.v, not below it
        (pt(2, 2), True),       # top edge: the bottom node lies below
        (pt(4, 2), True), (pt(0, 0), False), (pt(4, 0), False), (pt(0, 2), False),
        (pt(2, 1, 0.0), True), (pt(2, 1, 1.0), True),      # on the axis bounds
        (pt(2, 1, -1e-3), False), (pt(2, 1, 1.001), False),
    ]
    pts = np.stack([c[0] for c in cases])
    got = O.crop_mask(pts, axis, 0.0, 1.0, poly)
    assert got.tolist() == [c[1] for c in cases]


def test_oracle_voxel_means_against_brute_force():
    rng = np.random.default_rng(3)
    p = rng.normal(size=(3000, 3)).astype(np.float32)
    got = O.voxel_downsample(p, 0.4)
    org, dims, ijk = O.voxel_grid(p, 0.4)
    groups = {}
    for i, k in enumerate(map(tuple, ijk)):
        groups.setdefault(k, []).append(i)
    want = []
    for k in sorted(groups):
        s = np.zeros(3)
        for i in groups[k]:
            s = s + p[i].astype(np.float64)
        want.append((s / len(groups[k])).astype(np.float32))
    assert np.array_equal(got, np.array(want))


def test_oracle_nearest_against_brute_force():
    rng = np.random.default_rng(4)
    t = (rng.integers(-6, 6, (700, 3)) * 0.5).astype(np.float32)      # many exact ties
    q = np.concatenate([rng.normal(size=(300, 3)), rng.integers(-6, 6, (200, 3)) * 0.5 + 0.25])
    q = q.astype(np.float32)
    d, i = O.nearest(q, t, 0.6)
    d2 = O.exact_d2(q[:, None, :], t[None])
    best = d2.min(1)
    for k in range(len(q)):
        if best[k] < 0.36:
            j = np.nonzero(d2[k] == best[k])[0].min()
            assert i[k] == j and d[k] == np.sqrt(best[k])
        else:
            assert i[k] == -1 and d[k] == 0.6


def test_oracle_curve_is_numpy_histogram():
    d = np.array([0.0, 0.001, 0.0049, 0.00499, 0.005, 0.049, 0.0499, 0.05])
    c = O.curve(d, 0.01)
    assert len(c) == 499
    h, _ = np.histogram(d, np.arange(500) * 0.01 / 100)
    assert np.array_equal(c, np.cumsum(h) / len(d))


def test_uniform_downsample_keeps_every_kth():
    p = np.arange(30).reshape(10, 3).astype(np.float32)
    assert np.array_equal(O.uniform_downsample(p, 4), p[::2])
    assert np.array_equal(O.uniform_downsample(p, 10), p)


# ------------------------------------------------------------------------------ scene + CLI
def test_synthetic_scene_is_seeded(tmp_path):
    a = synth_tnt.make_scene(str(tmp_path / "a"), n_gt=2000, n_rec=2000, seed=3)
    b = synth_tnt.make_scene(str(tmp_path / "b"), n_gt=2000, n_rec=2000, seed=3)
    c = synth_tnt.make_scene(str(tmp_path / "c"), n_gt=2000, n_rec=2000, seed=4)
    for rel in ("rec.ply", "gt/Synth/Synth.ply", "gt/Synth/Synth_COLMAP_SfM.log",
                "gt/Synth/Synth_trans.txt", "run/view_names.txt", "run/cams/00000000_cam.txt"):
        assert (tmp_path / "a" / rel).read_bytes() == (tmp_path / "b" / rel).read_bytes(), rel
    assert (tmp_path / "a" / "rec.ply").read_bytes() != (tmp_path / "c" / "rec.ply").read_bytes()
    s = np.linalg.svd(a["rec_to_gt"][:3, :3], compute_uv=False)
    assert 1 / 3 - 1e-9 <= s[0] <= 1 / 0.3 + 1e-9 and np.ptp(s) < 1e-9
    traj = E.trajectory_from_run(a["run_dir"])
    assert len(traj) == 37 and len(E.read_log(os.path.join(
        a["gt_dir"], "Synth", "Synth_COLMAP_SfM.log"))) == 40


def test_cli_refusals_without_a_gpu(tmp_path):
    s = synth_tnt.make_scene(str(tmp_path), n_gt=1000, n_rec=1000, seed=0)
    base = ["--ply", s["ply"], "--run_dir", s["run_dir"], "--gt_dir", s["gt_dir"], "--scene", "Synth"]
    with pytest.raises(SystemExit, match="no tau for scene 'Synth'"):
        E.main(base)
    with pytest.raises(SystemExit, match="37 cameras and the ground-truth log 40"):
        E.main(base + ["--tau", "0.05"])
    with pytest.raises(SystemExit, match="ground truth"):
        E.main(["--ply", s["ply"], "--run_dir", s["run_dir"], "--gt_dir", s["gt_dir"], "--scene",
                "Barn"])
