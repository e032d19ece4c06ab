"""DTU scoring, CPU tier: the float64 oracle against brute force, the MATLAB conventions, PLY and
.mat I/O, and argument validation of the new entry points before any device work."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import dtu_eval_oracle as O

scipy_io = pytest.importorskip("scipy.io")


def _cloud(n, seed):
    """Clustered float32 points with exact duplicates: many neighbours within 0.2 mm."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(0, 3, (n // 20, 3))
    p = c[rng.integers(0, len(c), n)] + rng.normal(0, 0.15, (n, 3))
    p[: n // 10] = p[n // 2: n // 2 + n // 10]
    return (p + 500.0).astype(np.float32)


def _brute_d2(p):
    q = p.astype(np.float64)
    d = q[:, None, :] - q[None, :, :]
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_thinning_is_the_greedy_maximal_independent_set(seed):
    p = _cloud(1500, seed)
    dst = 0.2
    kept = O.thin(p, dst, seed)
    rank = np.empty(len(p), np.int64)
    rank[O.visiting_order(len(p), seed)] = np.arange(len(p))
    close = _brute_d2(p) <= dst * dst
    np.fill_diagonal(close, False)
    keep = np.zeros(len(p), bool)
    keep[kept] = True
    assert 0 < keep.sum() < len(p)
    assert not close[np.ix_(keep, keep)].any()                      # independent
    for i in np.nonzero(~keep)[0]:                                  # maximal, by a lower rank
        assert (close[i] & keep & (rank < rank[i])).any()
    # the sequential rule restated on the dense matrix
    ref = np.ones(len(p), bool)
    for i in O.visiting_order(len(p), seed):
        if ref[i]:
            ref[close[i]] = False
    assert np.array_equal(np.nonzero(ref)[0], kept)
    assert np.array_equal(O.thin(p, dst, seed), kept)               # seeded: repeatable


def test_oracle_capped_distance_grid_faces_and_cap():
    bb = np.array([[0.0, 0.0, 0.0], [130.0, 50.0, 10.0]])
    lo, hi = O.block_grid(bb)
    assert np.array_equal(lo, [0, 0, 0]) and np.array_equal(hi, [180, 60, 60])
    tgt = np.array([[10.0, 10.0, 10.0]], np.float32)
    q = np.array([[10, 10, 13],          # 3 mm away
                  [0, 10, 10],           # on the lower face: inside
                  [180, 10, 10],         # on the upper face: outside -> 60
                  [-1e-3, 10, 10],       # below BB1 -> 60
                  [10, 10, 70 - 1e-4],   # beyond the cap within the grid... z >= 60: outside
                  [70, 10, 10],          # exactly 60 mm away -> 60
                  [69, 10, 10],          # 59 mm
                  [100, 10, 10]], np.float32)
    d = O.capped_nn(q, tgt, bb)
    assert d[0] == pytest.approx(3.0)
    assert d[1] == pytest.approx(10.0)
    assert d[2] == 60.0 and d[3] == 60.0 and d[4] == 60.0
    assert d[5] == 60.0 and d[6] == pytest.approx(59.0) and d[7] == 60.0
    assert np.all(O.capped_nn(q, np.zeros((0, 3), np.float32), bb) == 60.0)


def test_matlab_round_and_mask_index():
    from casmvsnet_pl_b200 import dtu_eval
    x = np.array([0.5, 1.5, 2.5, -0.5, -1.5, 2.4999999999999996, 0.49999999999999994, 3.0])
    want = np.array([1, 2, 3, -1, -2, 2, 0, 3], np.float64)
    assert np.array_equal(O.matlab_round(x), want)
    assert np.array_equal(dtu_eval.round_half_away(torch.from_numpy(x)).numpy(), want)
    mask = np.zeros((3, 3, 3), bool)
    mask[1, 0, 0] = True                              # MATLAB index (2,1,1)
    bb = np.array([[0.0, 0.0, 0.0], [2.0, 2.0, 2.0]])
    pts = np.array([[0.5, 0, 0],                      # (0.5 + 1) -> round 1.5 = 2: inside
                    [0.49, 0, 0],                     # -> 1: outside the mask
                    [-0.5, 0, 0],                     # -> 0.5 -> 1 (half away): index 1
                    [-0.51, 0, 0],                    # -> 0: outside the grid
                    [2.49, 0, 0]], np.float32)        # -> 3.49 -> 3: in grid, not masked
    assert O.data_in_mask(pts, mask, bb, 1.0).tolist() == [True, False, False, False, False]
    assert O.data_in_mask(pts - 1, mask, bb - 1, 1.0).tolist() == [True, False, False, False, False]


def test_statistics_follow_matlab():
    from casmvsnet_pl_b200 import dtu_eval
    d = np.array([1.0, 4.0, 2.0, 30.0, 3.0, 19.999, 20.0])
    sel = np.array([True, True, True, True, True, False, True])
    s = O.stats(d, sel)
    assert s["n"] == 4 and s["mean"] == 2.5 and s["median"] == 2.5
    assert s["var"] == pytest.approx(np.var([1, 4, 2, 3], ddof=1))
    t = dtu_eval.matlab_stats(torch.from_numpy(d), torch.from_numpy(sel))
    assert t == pytest.approx(s)
    one = dtu_eval.matlab_stats(torch.tensor([5.0]), torch.tensor([True]))
    assert one["var"] == 0.0 and one["median"] == 5.0 and O.stats([5.0], [True])["var"] == 0.0
    none = dtu_eval.matlab_stats(torch.tensor([25.0]), torch.tensor([True]))
    assert none["n"] == 0 and np.isnan(none["mean"]) and np.isnan(O.stats([25.0], [True])["mean"])
    odd = dtu_eval.matlab_stats(torch.tensor([3.0, 1.0, 2.0]), torch.ones(3, dtype=torch.bool))
    assert odd["median"] == 2.0
    s2 = dtu_eval.summarize([dict(scan=1, acc=1.0, comp=3.0), dict(scan=4, acc=2.0, comp=5.0)])
    assert (s2["acc"], s2["comp"], s2["overall"], s2["scans"]) == (1.5, 4.0, 2.75, [1, 4])


def test_plane_test_and_block_grid_match_oracle():
    from casmvsnet_pl_b200 import dtu_eval
    bb = np.array([[-3.7, 1.1, 400.3], [151.2, 60.0, 700.9]])
    lo, hi = dtu_eval.block_grid(bb)
    olo, ohi = O.block_grid(bb)
    assert np.array_equal(lo, olo) and np.array_equal(hi, ohi)
    assert dtu_eval.scan_number("scan23") == 23 and dtu_eval.scan_number("/x/scan9.ply") == 9
    with pytest.raises(ValueError):
        dtu_eval.scan_number("scene")


def test_read_ply_round_trips_write_ply(tmp_path):
    from casmvsnet_pl_b200 import fusion, io
    rng = np.random.default_rng(0)
    xyz = rng.normal(0, 100, (257, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (257, 3)).astype(np.uint8)
    fusion.write_ply(tmp_path / "a.ply", xyz, rgb)
    v = io.read_ply(tmp_path / "a.ply")
    assert v.dtype.names == ("x", "y", "z", "red", "green", "blue")
    assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], 1), xyz)
    assert np.array_equal(np.stack([v["red"], v["green"], v["blue"]], 1), rgb)
    fusion.write_ply(tmp_path / "e.ply", np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8))
    assert len(io.read_ply(tmp_path / "e.ply")) == 0


def test_read_ply_ascii_and_binary_with_faces(tmp_path):
    from casmvsnet_pl_b200 import io
    from casmvsnet_pl_b200.dtu_eval import read_points
    (tmp_path / "a.ply").write_text(
        "ply\nformat ascii 1.0\ncomment hand written\nelement vertex 3\nproperty float x\n"
        "property float y\nproperty float z\nproperty uchar red\nelement face 1\n"
        "property list uchar int vertex_indices\nend_header\n"
        "1.5 -2 3e2 7\n0 0 0 255\n-0.25 1 2 0\n3 0 1 2\n")
    v = io.read_ply(tmp_path / "a.ply")
    assert v["x"].tolist() == [1.5, 0.0, -0.25] and v["z"][0] == 300.0 and v["red"].tolist() == [7, 255, 0]
    assert read_points(tmp_path / "a.ply").dtype == np.float32
    dt = np.dtype([("x", "<f4"), ("nx", "<f4"), ("y", "<f4"), ("z", "<f4"), ("q", "<f8"), ("i", "<i4")])
    verts = np.zeros(4, dt)
    verts["x"], verts["y"], verts["z"] = [1, 2, 3, 4], [5, 6, 7, 8], [9, 10, 11, 12]
    verts["q"] = 0.5
    head = ("ply\nformat binary_little_endian 1.0\nelement vertex 4\nproperty float x\n"
            "property float nx\nproperty float y\nproperty float z\nproperty double q\n"
            "property int i\nelement face 2\nproperty list uchar int vertex_indices\nend_header\n")
    faces = bytes([3]) + np.array([0, 1, 2], "<i4").tobytes() + bytes([3]) + np.array([1, 2, 3], "<i4").tobytes()
    (tmp_path / "b.ply").write_bytes(head.encode() + verts.tobytes() + faces)
    p = read_points(tmp_path / "b.ply")
    assert p.tolist() == [[1, 5, 9], [2, 6, 10], [3, 7, 11], [4, 8, 12]]
    assert io.read_ply(tmp_path / "b.ply")["q"].tolist() == [0.5] * 4
    for bad in (head.replace("binary_little_endian", "binary_big_endian"),
                head.replace("property float nx\n", "property list uchar float nx\n"),
                head.replace("element vertex 4\n", "element face 2\nproperty list uchar int v\n"
                             "element vertex 4\n", 1),
                "plx\n" + head[4:]):
        (tmp_path / "bad.ply").write_bytes(bad.encode() + verts.tobytes())
        with pytest.raises(ValueError):
            io.read_ply(tmp_path / "bad.ply")
    (tmp_path / "short.ply").write_bytes(head.encode() + verts.tobytes()[:40])
    with pytest.raises(ValueError):
        io.read_ply(tmp_path / "short.ply")


def test_mat_ground_truth_loads_back(tmp_path):
    from casmvsnet_pl_b200 import dtu_eval, synth_dtu
    stl = np.array([[0, 0, 0], [5, 5, 5], [12.5, 3, 1]], np.float32)
    bb = synth_dtu.write_ground_truth(str(tmp_path), 9, stl, ground_z=1.0)
    mask, bb2, res = dtu_eval.load_obs_mask(str(tmp_path), 9)
    assert np.array_equal(bb2, bb) and res == 1.0 and mask.dtype == bool
    assert mask.shape == tuple(np.floor((bb[1] - bb[0]) / res).astype(int) + 1)
    assert mask[10, 10, 10] and not mask[0, 0, 0]                 # (0,0,0) is 10 voxels in
    assert np.array_equal(dtu_eval.load_plane(str(tmp_path), 9), [0, 0, 1, -1])
    assert np.array_equal(dtu_eval.read_points(dtu_eval.stl_path(str(tmp_path), 9)), stl)
    # axis order is kept as stored
    m = np.zeros((2, 3, 4), bool)
    m[1, 2, 3] = True
    scipy_io.savemat(tmp_path / "m.mat", {"ObsMask": m})
    back = scipy_io.loadmat(tmp_path / "m.mat")["ObsMask"]
    assert back.shape == (2, 3, 4) and back.astype(bool)[1, 2, 3] and back.sum() == 1


def test_new_entry_points_reject_bad_arguments(tmp_path):
    """Validation comes before any device work (no GPU here)."""
    from casmvsnet_pl_b200 import _lib, dtu_eval
    lib = _lib.load()
    one = ctypes.c_void_p(16)
    assert lib.casmvs_pcd_cell_keys(None, 0, 0.0, 0.0, 0.0, 0.2, 4, 4, 4, 1, None, None) == 0
    assert lib.casmvs_pcd_cell_keys(one, 5, 0.0, 0.0, 0.0, 0.2, 4, 4, 4, 3, one, None) < 0
    assert b"sub" in lib.casmvs_last_error()
    assert lib.casmvs_pcd_cell_keys(one, 5, 0.0, 0.0, 0.0, 0.0, 4, 4, 4, 1, one, None) < 0
    assert lib.casmvs_pcd_cell_keys(one, 5, 0.0, 0.0, 0.0, 0.2, 4, 1 << 20, 4, 1, one, None) < 0
    assert lib.casmvs_pcd_cell_keys(None, 5, 0.0, 0.0, 0.0, 0.2, 4, 4, 4, 1, one, None) < 0
    assert b"null" in lib.casmvs_last_error()
    need = lib.casmvs_pcd_thin_workspace_bytes(100, 10)
    assert need >= 100 * 4 + 27 * 10 * 4
    assert lib.casmvs_pcd_thin_prepare(one, one, 100, 10, 4, 4, 4, one, need - 1, None) < 0
    assert b"workspace" in lib.casmvs_last_error()
    assert lib.casmvs_pcd_thin_prepare(one, one, 5, 10, 4, 4, 4, one, 1 << 20, None) < 0
    assert lib.casmvs_pcd_thin_round(one, one, one, 100, 10, -1.0, one, one, one, need, None) < 0
    assert lib.casmvs_pcd_thin_round(one, one, one, 100, 10, 0.2, one, None, one, need, None) < 0
    d3 = (ctypes.c_double * 3)(0, 0, 0)
    i3 = (ctypes.c_int * 3)(4, 4, 4)
    assert lib.casmvs_pcd_capped_nn(one, 4, one, one, one, 1, one, d3, 0.0, i3, d3, d3, 60.0,
                                    one, None) < 0
    assert lib.casmvs_pcd_capped_nn(one, 4, one, one, one, 1, one, None, 1.0, i3, d3, d3, 60.0,
                                    one, None) < 0
    assert lib.casmvs_pcd_capped_nn(one, 4, None, one, one, 1, one, d3, 1.0, i3, d3, d3, 60.0,
                                    one, None) < 0
    # Python surface: checked before anything touches a device
    with pytest.raises(ValueError):
        dtu_eval.thin(torch.zeros(4, 3))                             # CPU tensor
    with pytest.raises(ValueError):
        dtu_eval.capped_nn(torch.zeros(4, 2), torch.zeros(4, 3), [0] * 3, [1] * 3)
    with pytest.raises(ValueError):
        dtu_eval.evaluate_scan(torch.zeros(4, 3), 1, str(tmp_path))  # CPU tensor
    with pytest.raises(ValueError):
        dtu_eval.evaluate_scan(str(tmp_path / "x.ply"), "one", str(tmp_path))
    with pytest.raises(ValueError):
        dtu_eval.evaluate_scan(str(tmp_path / "x.ply"), 1, str(tmp_path), dst=0.0)
    with pytest.raises(FileNotFoundError):
        dtu_eval.evaluate_scan(str(tmp_path / "x.ply"), 1, str(tmp_path / "missing"))
    with pytest.raises(TypeError):
        dtu_eval.evaluate_scan(np.zeros((4, 3), np.float32), 1, str(tmp_path))
    with pytest.raises(ValueError):
        dtu_eval.summarize([])


def test_synthetic_scene_is_seeded(tmp_path):
    from casmvsnet_pl_b200 import synth_dtu
    a = synth_dtu.make_scene(str(tmp_path / "a"), 3, n_stl=2000, n_data=3000, seed=5)
    b = synth_dtu.make_scene(str(tmp_path / "b"), 3, n_stl=2000, n_data=3000, seed=5)
    assert a.shape == (3000, 3) and a.dtype == np.float32 and np.array_equal(a, b)
    assert len(np.unique(a, axis=0)) < len(a)                        # exact duplicates
    from casmvsnet_pl_b200.dtu_eval import load_obs_mask
    _, bb, _ = load_obs_mask(str(tmp_path / "a"), 3)
    assert ((a < bb[0]) | (a > bb[1])).any(1).sum() > 0            # outliers beyond BB
