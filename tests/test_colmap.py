"""COLMAP scene conversion, CPU tier: the model readers (binary and text), their validation, the
float64 view-selection oracle on hand-computed cases, source ranking, the skip rule, the depth
range picks, the written record of a run, the per-data-set --depth_interval default and the
argument checks of the new C entries."""
import ctypes
import math
import os

import numpy as np
import pytest

from casmvsnet_pl_b200 import colmap, io as cio, synth_scenes
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import view_select_oracle as O


def _same_model(a, b):
    assert a.cameras.keys() == b.cameras.keys()
    for k in a.cameras:
        assert a.cameras[k][:3] == b.cameras[k][:3]
        assert np.array_equal(a.cameras[k][3], b.cameras[k][3])
    assert a.images.keys() == b.images.keys()
    for k in a.images:
        qa, ta, ca, na = a.images[k]
        qb, tb, cb, nb = b.images[k]
        assert np.array_equal(qa, qb) and np.array_equal(ta, tb) and ca == cb and na == nb
    assert np.array_equal(a.point_ids, b.point_ids)
    assert np.array_equal(a.xyz, b.xyz)
    assert np.array_equal(a.track_ptr, b.track_ptr)
    assert np.array_equal(a.track_img, b.track_img)


@pytest.mark.parametrize("fmt", ["bin", "txt"])
def test_reader_round_trips_the_synthetic_model(tmp_path, fmt):
    model = synth_scenes.colmap_model(n_views=6, n_points=400, seed=1)
    colmap.write_model(str(tmp_path), model, fmt)
    _same_model(colmap.read_model(str(tmp_path)), model)


def test_both_formats_read_the_same(tmp_path):
    model = synth_scenes.make_colmap(str(tmp_path), n_views=5, image_wh=(64, 48), n_points=300,
                                     seed=2, fmt="both")
    sparse = colmap.find_sparse_dir(str(tmp_path))
    _same_model(colmap.read_model(sparse, ".bin"), colmap.read_model(sparse, ".txt"))
    _same_model(colmap.read_model(sparse), model)
    names = sorted(os.listdir(tmp_path / "images"))
    assert names == sorted(im[3] for im in model.images.values())
    from PIL import Image
    for q, t, cid, name in model.images.values():           # each view at its camera's size
        assert Image.open(tmp_path / "images" / name).size == tuple(model.cameras[cid][1:3])


def test_scene_views_poses_and_tracks():
    model = synth_scenes.colmap_model(n_views=6, n_points=300, seed=3, n_single=5, n_dup=7)
    sc = colmap.Scene(model)
    assert sc.names == sorted(im[3] for im in model.images.values())
    by_name = {im[3]: iid for iid, im in model.images.items()}
    for v, name in enumerate(sc.names):
        q, t, cid, _ = model.images[by_name[name]]
        cam = model.cameras[cid]
        assert np.allclose(sc.E[v, :3, :3], colmap.qvec_to_rotmat(q)) and np.array_equal(sc.E[v, :3, 3], t)
        assert np.allclose(sc.centres[v], -colmap.qvec_to_rotmat(q).T @ t)
        assert tuple(sc.wh[v]) == cam[1:3]
        if cam[0] == "SIMPLE_PINHOLE":
            assert sc.K[v, 0, 0] == sc.K[v, 1, 1] == cam[3][0]
        else:
            assert (sc.K[v, 0, 0], sc.K[v, 1, 1], sc.K[v, 0, 2], sc.K[v, 1, 2]) == tuple(cam[3])
    vid = {by_name[n]: v for v, n in enumerate(sc.names)}
    n_dup = 0
    for p in range(len(model.xyz)):
        raw = [vid[int(i)] for i in model.track_img[model.track_ptr[p]:model.track_ptr[p + 1]]]
        got = sc.track_img[sc.track_ptr[p]:sc.track_ptr[p + 1]].tolist()
        assert got == sorted(set(raw))                      # an image listed twice counts once
        n_dup += len(raw) != len(got)
    assert n_dup == 7
    assert int(np.sum(np.diff(sc.track_ptr) == 1)) >= 5


def test_rotation_quaternion_round_trip():
    rng = np.random.default_rng(0)
    for _ in range(20):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        q = -q if q[0] < 0 else q
        R = colmap.qvec_to_rotmat(q)
        assert np.allclose(R @ R.T, np.eye(3)) and np.isclose(np.linalg.det(R), 1)
        assert np.allclose(colmap.rotmat_to_qvec(R), q)


@pytest.mark.parametrize("fmt", ["bin", "txt"])
def test_distorted_camera_model_is_rejected_by_name(tmp_path, fmt):
    model = synth_scenes.colmap_model(n_views=4, n_points=100, seed=4)
    model.cameras[2] = ("OPENCV", 200, 150, np.array([200.0, 200.0, 100.0, 75.0, 0.1, 0.01, 0, 0]))
    colmap.write_model(str(tmp_path), model, fmt)
    with pytest.raises(ValueError, match="OPENCV.*image_undistorter"):
        colmap.read_model(str(tmp_path))


@pytest.mark.parametrize("fmt", ["bin", "txt"])
def test_bad_track_ids_are_rejected(tmp_path, fmt):
    model = synth_scenes.colmap_model(n_views=4, n_points=100, seed=5)
    model.track_img[7] = 999
    colmap.write_model(str(tmp_path), model, fmt)
    with pytest.raises(ValueError, match="image 999"):
        colmap.read_model(str(tmp_path))


def test_non_finite_values_are_rejected():
    model = synth_scenes.colmap_model(n_views=4, n_points=100, seed=6)
    model.xyz[3, 1] = np.nan
    with pytest.raises(ValueError, match="not finite"):
        colmap.check_model(model)
    model = synth_scenes.colmap_model(n_views=4, n_points=100, seed=6)
    iid = next(iter(model.images))
    q, t, cid, name = model.images[iid]
    model.images[iid] = (q, np.array([0, np.inf, 0]), cid, name)
    with pytest.raises(ValueError, match="not finite"):
        colmap.check_model(model)
    model = synth_scenes.colmap_model(n_views=4, n_points=100, seed=6)
    model.images[iid] = (q, t, 77, name)
    with pytest.raises(ValueError, match="camera 77"):
        colmap.check_model(model)


def _three_cameras():
    """Cameras at unit distance from the origin at 0, 5 and 15 degrees about the y axis."""
    a = np.deg2rad([0.0, 5.0, 15.0])
    return np.stack([np.sin(a), np.zeros(3), np.cos(a)], 1)


def test_oracle_scores_hand_computed_case():
    c = _three_cameras()
    xyz = np.zeros((2, 3))
    ptr = np.array([0, 3, 5])
    img = np.array([0, 1, 2, 1, 2])          # point 0 seen by all three, point 1 by views 1 and 2
    want = np.zeros((3, 3))
    want[0, 1] = 1.0                         # theta = 5 -> G = 1
    want[0, 2] = math.exp(-0.5)              # theta = 15 -> exp(-(10)^2 / 200)
    want[1, 2] = 2 * math.exp(-25 / 200)     # theta = 10, twice
    want = want + want.T
    for f in (O.view_scores, O.view_scores_vec):
        assert np.allclose(f(c, xyz, ptr, img, 3), want, rtol=1e-14, atol=1e-15)
    assert math.isclose(float(O.weight(4.0)), math.exp(-0.5), rel_tol=1e-15)
    assert float(O.weight(5.0)) == 1.0


def test_oracle_vectorised_equals_loop_on_ragged_tracks():
    c, xyz, ptr, img = synth_scenes.sparse_tracks(30, 300, (1, 25), seed=7)
    assert np.array_equal(O.view_scores(c, xyz, ptr, img, 30), O.view_scores_vec(c, xyz, ptr, img, 30))


def test_source_ranking_and_tie_rule():
    s = np.array([[0, 3, 5, 3, 0, 1],
                  [3, 0, 2, 2, 2, 0],
                  [5, 2, 0, 0, 0, 0],
                  [3, 2, 0, 0, 4, 0],
                  [0, 2, 0, 4, 0, 0],
                  [1, 0, 0, 0, 0, 0]], np.float64)
    want = [[2, 1, 3, 5], [0, 2, 3, 4], [0, 1], [4, 0, 1], [3, 1], [0]]
    got = colmap.select_sources(s)
    assert [[j for j, _ in r] for r in got] == want
    assert got[0][0] == (2, 5.0)
    assert O.select_sources(s) == want
    assert [[j for j, _ in r] for r in colmap.select_sources(s, n_src=2)] == [r[:2] for r in want]


def test_skip_rule():
    s = np.zeros((5, 5))
    s[0, 1:] = s[1:, 0] = 1.0
    s[1, 2] = s[2, 1] = s[1, 3] = s[3, 1] = 0.5
    count = np.array([100, 100, 100, 19, 20])
    q = np.tile([[2.0, 4.0]], (5, 1))
    sources, refs, skipped, dmin, dmax = colmap.assemble(s, count, q, n_views=3)
    # view 0: 4 sources; 1: 3; 2: 2; 3: 2 sources but 19 points; 4: 1 source
    assert refs == [0, 1, 2] and sorted(skipped) == [3, 4]
    assert "19" in skipped[3] and "1 valid sources" in skipped[4]
    for v in range(5):
        n_src = len(sources[v])
        assert O.skipped(n_src, count[v], 3) == (v in skipped)
    assert np.all(dmin == 1.5) and np.all(dmax == 5.0)


def test_depth_range_picks():
    """z = 1 .. 150 in view 0's camera (shuffled, plus points behind it and points of view 1):
    q(0.01) = z[floor(1.49)] = 2, q(0.99) = z[floor(147.51)] = 148."""
    rng = np.random.default_rng(8)
    z0 = rng.permutation(np.arange(1, 151).astype(np.float64))
    xyz = np.concatenate([np.stack([0 * z0, 0 * z0, z0], 1), [[0, 0, -3.0], [0, 0, -1.0]],
                          [[0, 0, 7.0]]])
    E = np.tile(np.eye(4), (2, 1, 1))
    E[1, 2, 3] = 10.0                                       # view 1: z = Z + 10
    ptr = np.arange(len(xyz) + 1)
    img = np.zeros(len(xyz), np.int64)
    img[-1] = 1
    count, q = colmap.depth_stats(E, xyz, ptr, img, device="cpu")
    assert count.tolist() == [150, 1]
    assert q[0].tolist() == [2.0, 148.0] and q[1].tolist() == [17.0, 17.0]
    n, dmin, dmax = O.depth_range(E, xyz, ptr, img, 0)
    assert (n, dmin, dmax) == (150, 1.5, 185.0)
    _, _, _, dmin, dmax = colmap.assemble(np.zeros((2, 2)), count, q, 2)
    assert dmin[0] == 1.5 and dmax[0] == 185.0
    count, q = colmap.depth_stats(E, xyz[:0], np.zeros(1, np.int64), img[:0], device="cpu")
    assert count.tolist() == [0, 0] and np.isnan(q).all()


def test_written_cams_and_pair_read_back_unchanged(tmp_path):
    model = synth_scenes.colmap_model(n_views=5, n_points=200, seed=9)
    sc = colmap.Scene(model)
    E32, K32 = sc.E.astype(np.float32), sc.K.astype(np.float32)
    rng = np.random.default_rng(0)
    rngs = {v: (float(np.float32(rng.uniform(1, 2))), float(np.float32(rng.uniform(0, 0.01))),
                float(rng.uniform(3, 4))) for v in range(len(sc))}
    colmap.write_cams(str(tmp_path / "cams"), E32, K32, rngs, 192.0)
    for v in range(len(sc)):
        K, E, dmin = cio.read_cam_file(str(tmp_path / "cams" / f"{v:08d}_cam.txt"))
        assert np.array_equal(K, K32[v]) and np.array_equal(E, E32[v]) and dmin == rngs[v][0]
        last = open(tmp_path / "cams" / f"{v:08d}_cam.txt").read().splitlines()[-1].split()
        assert float(last[1]) == rngs[v][1] and last[2] == "192" and float(last[3]) == rngs[v][2]
    metas = [(0, [(2, 3.25), (1, 0.1 + 0.2)]), (3, [(4, 1e-3), (0, 1e-300), (1, 5e-324)])]
    colmap.write_pair(str(tmp_path / "pair.txt"), metas)
    assert cio.read_pair_file(str(tmp_path / "pair.txt")) == [(r, [s for s, _ in ss]) for r, ss in metas]
    toks = open(tmp_path / "pair.txt").read().split()
    assert toks[:5] == ["2", "0", "2", "2", "3.25"] and float(toks[6]) == 0.1 + 0.2                     # scores are written exactly


def test_depth_interval_default_is_resolved_per_dataset(tmp_path):
    r = ["--root_dir", str(tmp_path)]
    for ds in ("dtu", "tanks", "blendedmvs"):
        assert ep.parse_args(r + ["--dataset_name", ds]).depth_interval == 2.65
        assert ep.parse_args(r + ["--dataset_name", ds, "--depth_interval", "3.5"]).depth_interval == 3.5
    assert ep.parse_args(r).depth_interval == 2.65                     # dtu is the default data set
    assert ep.parse_args(r + ["--dataset_name", "colmap"]).depth_interval == 192.0
    assert ep.parse_args(r + ["--dataset_name", "colmap", "--depth_interval", "96"]).depth_interval == 96.0
    assert ep.parse_args(r + ["--dataset_name", "colmap"]).out_dir == os.path.join("results", "colmap")


def test_view_scores_entries_validate_before_any_cuda_call():
    from casmvsnet_pl_b200 import _lib
    lib = _lib.load()
    one = ctypes.c_void_p(256)
    rc = lib.casmvs_view_scores_fwd(one, one, one, one, -1, 10, one, one, 1 << 30, None)
    assert rc < 0 and b"bad dims" in lib.casmvs_last_error()
    rc = lib.casmvs_view_scores_fwd(one, one, one, one, 70000, 10, one, one, 1 << 30, None)
    assert rc < 0 and b"bad dims" in lib.casmvs_last_error()
    rc = lib.casmvs_view_scores_fwd(one, one, one, one, 4, -2, one, one, 1 << 30, None)
    assert rc < 0 and b"bad dims" in lib.casmvs_last_error()
    rc = lib.casmvs_view_scores_fwd(one, one, one, one, 4, 10, None, one, 1 << 30, None)
    assert rc < 0 and b"null" in lib.casmvs_last_error()
    rc = lib.casmvs_view_scores_fwd(None, one, one, one, 4, 10, one, one, 1 << 30, None)
    assert rc < 0 and b"null" in lib.casmvs_last_error()
    rc = lib.casmvs_view_scores_fwd(one, one, one, None, 4, 10, one, one, 1 << 30, None)
    assert rc < 0 and b"null" in lib.casmvs_last_error()
    rc = lib.casmvs_view_scores_fwd(one, one, one, one, 4, 10, one, ctypes.c_void_p(264), 1 << 30, None)
    assert rc < 0 and b"workspace must be 256-byte aligned" in lib.casmvs_last_error()
    rc = lib.casmvs_view_scores_fwd(one, ctypes.c_void_p(260), one, one, 4, 10, one, one, 1 << 30, None)
    assert rc < 0 and b"points must be 8-byte aligned" in lib.casmvs_last_error()
    assert lib.casmvs_view_scores_fwd(None, None, None, None, 0, 10, None, None, 0, None) == 0
    assert lib.casmvs_view_scores_workspace_bytes(1, 10, 0) == 0
    assert lib.casmvs_view_scores_workspace_bytes(4, 0, 0) == 0
    assert lib.casmvs_view_scores_workspace_bytes(70000, 10, 0) == 0
