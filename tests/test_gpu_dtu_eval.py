"""DTU scoring on the GPU against the float64 oracle (oracle/dtu_eval_oracle.py) on seeded
synthetic scenes of 100k-300k points: thinning, capped distances, masks and statistics."""
import json
import math

import numpy as np
import pytest
import torch

from oracle import dtu_eval_oracle as O

pytestmark = pytest.mark.gpu


def _oracle_inputs(gt, scan):
    from casmvsnet_pl_b200 import dtu_eval
    obs, bb, res = dtu_eval.load_obs_mask(gt, scan)
    return (dtu_eval.read_points(dtu_eval.stl_path(gt, scan)), obs, bb, res,
            dtu_eval.load_plane(gt, scan))


def _close_to_threshold(d, thr=20.0, tol=1e-5):
    return np.abs(np.asarray(d) - thr) <= tol


def _compare(got, want, data, stl):
    assert np.array_equal(got["kept"].cpu().numpy(), want["kept"])
    dd, ds = got["Ddata"].cpu().numpy(), got["Dstl"].cpu().numpy()
    for g, w in ((dd, want["Ddata"]), (ds, want["Dstl"])):
        below = w < 60.0
        assert np.abs(g[below] - w[below]).max(initial=0.0) <= 1e-5
        assert np.all(g[~below] == 60.0)
    assert np.array_equal(got["data_in_mask"].cpu().numpy(), want["data_in_mask"])
    assert np.array_equal(got["stl_above_plane"].cpu().numpy(), want["stl_above_plane"])
    for side, d_w, sel in (("acc", want["Ddata"], want["data_in_mask"]),
                           ("comp", want["Dstl"], want["stl_above_plane"])):
        w = want[side]
        n_edge = int((sel & _close_to_threshold(d_w)).sum())
        assert abs(got[f"n_{side}"] - w["n"]) <= n_edge
        if w["n"] == 0:
            assert got[f"n_{side}"] == 0 and math.isnan(got[side])
            continue
        if n_edge == 0:
            assert got[side] == pytest.approx(w["mean"], rel=1e-6)
            assert got[f"{side}_median"] == pytest.approx(w["median"], rel=1e-6)
            assert got[f"{side}_var"] == pytest.approx(w["var"], rel=1e-5)


@pytest.mark.parametrize("seed,n_stl,n_data", [(0, 100_000, 150_000), (1, 120_000, 300_000),
                                               (2, 60_000, 200_000)])
def test_scores_match_oracle_on_synthetic_scenes(tmp_path, seed, n_stl, n_data):
    from casmvsnet_pl_b200 import dtu_eval, synth_dtu
    gt = str(tmp_path / "gt")
    data = synth_dtu.make_scene(gt, 4, n_stl, n_data, seed=seed)
    got = dtu_eval.evaluate_scan(torch.from_numpy(data).cuda(), 4, gt, seed=seed, return_arrays=True)
    stl, obs, bb, res, plane = _oracle_inputs(gt, 4)
    want = O.evaluate(data, stl, obs, bb, res, plane, 0.2, seed)
    assert 0 < len(want["kept"]) < len(data)
    assert want["acc"]["n"] > 1000 and want["comp"]["n"] > 1000
    assert (want["Dstl"] > 1.0).sum() > 100                       # the missed disc is scored
    _compare(got, want, data, stl)
    assert got["overall"] == pytest.approx((got["acc"] + got["comp"]) / 2)


def test_edge_cases_match_oracle(tmp_path):
    """Empty mask, empty data cloud, all data outside the block grid, a cloud of duplicates."""
    from casmvsnet_pl_b200 import dtu_eval, synth_dtu
    gt = str(tmp_path / "gt")
    data = synth_dtu.make_scene(gt, 1, 50_000, 100_000, seed=7, empty_mask=True)
    stl, obs, bb, res, plane = _oracle_inputs(gt, 1)
    assert not obs.any()
    lo, hi = dtu_eval.block_grid(bb)
    cases = {
        "empty_mask": data,
        "empty": np.zeros((0, 3), np.float32),
        "outside": data[:20_000] + np.array([hi[0] + 5.0 - data[:20_000, 0].min(), 0, 0], np.float32),
        "duplicates": np.repeat(data[:2_000], 50, axis=0),
    }
    for name, pts in cases.items():
        got = dtu_eval.evaluate_scan(torch.from_numpy(pts).cuda(), 1, gt, seed=3, return_arrays=True)
        want = O.evaluate(pts, stl, obs, bb, res, plane, 0.2, 3)
        _compare(got, want, pts, stl)
        assert got["n_acc"] == 0 and math.isnan(got["acc"]), name      # nothing in the mask
        if name == "empty":
            assert np.all(got["Dstl"].cpu().numpy() == 60.0), name
        if name == "outside":
            assert np.all(got["Ddata"].cpu().numpy() == 60.0), name
    got = dtu_eval.evaluate_scan(torch.from_numpy(cases["duplicates"]).cuda(), 1, gt, seed=3)
    assert got["n_thinned"] <= 2_000


def test_same_seed_is_bit_identical_and_seed_changes_the_set(tmp_path):
    from casmvsnet_pl_b200 import dtu_eval, synth_dtu
    gt = str(tmp_path / "gt")
    data = torch.from_numpy(synth_dtu.make_scene(gt, 2, 80_000, 200_000, seed=11)).cuda()
    a = dtu_eval.evaluate_scan(data, 2, gt, seed=5, return_arrays=True)
    b = dtu_eval.evaluate_scan(data, 2, gt, seed=5, return_arrays=True)
    c = dtu_eval.evaluate_scan(data, 2, gt, seed=6, return_arrays=True)
    for k in ("kept", "Ddata", "Dstl", "data_in_mask", "stl_above_plane"):
        assert torch.equal(a[k], b[k]), k
    for k in ("acc", "comp", "overall", "acc_median", "comp_median", "acc_var", "comp_var"):
        assert a[k] == b[k], k
    assert not torch.equal(a["kept"], c["kept"])
    assert a["acc"] == pytest.approx(c["acc"], rel=0.05)


def test_nearest_neighbour_far_and_face_queries():
    """Queries far from every target, on the grid faces and at the cap, brute-forced."""
    from casmvsnet_pl_b200 import dtu_eval
    rng = np.random.default_rng(0)
    bb = np.array([[0.0, 0.0, 0.0], [200.0, 100.0, 80.0]])
    lo, hi = dtu_eval.block_grid(bb)
    tgt = np.concatenate([rng.uniform(0, 20, (20_000, 3)), rng.uniform(150, 160, (500, 3))]).astype(np.float32)
    q = rng.uniform([-30, -30, -30], [250, 130, 130], (30_000, 3)).astype(np.float32)
    q[:3] = [[0, 0, 0], [hi[0], 5, 5], [80, 10, 10]]
    got = dtu_eval.capped_nn(torch.from_numpy(q).cuda(), torch.from_numpy(tgt).cuda(), lo, hi).cpu().numpy()
    want = O.capped_nn(q, tgt, bb)
    below = want < 60
    assert below.sum() > 500 and (~below).sum() > 500
    assert np.abs(got[below] - want[below]).max() <= 1e-5 and np.all(got[~below] == 60.0)


def test_run_scan_scores_fused_cloud_like_evaluate_scan(tmp_path):
    """eval_pipeline with scoring on: scores of fuse_scan's CUDA tensor == evaluate_scan on the
    returned points == evaluate_scan on the PLY written from them."""
    cv2 = pytest.importorskip("cv2")
    from casmvsnet_pl_b200 import ABN, dtu_eval, eval_pipeline, synth, synth_dtu
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    root = tmp_path / "dtu"
    (root / "Cameras").mkdir(parents=True)
    (root / "Rectified" / "scan7").mkdir(parents=True)
    rng = np.random.default_rng(0)
    W, H, n = 160, 128, 4
    K4 = synth.intrinsics(0, W, H)
    for vid in range(n):
        t = np.deg2rad(3.0 * vid)
        E = np.eye(4)
        E[:3, :3] = [[np.cos(t), 0, np.sin(t)], [0, 1, 0], [-np.sin(t), 0, np.cos(t)]]
        E[:3, 3] = [-680 * np.sin(t), 0, 680 * (1 - np.cos(t))]
        rows = ["extrinsic"] + [" ".join(f"{v:.6f}" for v in r) for r in E] + ["", "intrinsic"]
        rows += [" ".join(f"{v:.6f}" for v in r) for r in K4] + ["", "425.0 2.65"]
        (root / "Cameras" / f"{vid:08d}_cam.txt").write_text("\n".join(rows) + "\n")
        cv2.imwrite(str(root / "Rectified" / "scan7" / f"rect_{vid + 1:03d}_3_r5000.png"),
                    rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
    (root / "Cameras" / "pair.txt").write_text(
        "4\n0\n3 1 9.0 2 8.0 3 7.0\n1\n3 0 9.0 2 8.0 3 7.0\n2\n3 1 9.0 3 8.0 0 7.0\n3\n3 2 9.0 1 8.0 0 7.0\n")
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN, precision="tf32")
    synth.randomize_model_(model, 0)
    model = model.eval().cuda()
    scan = eval_pipeline.DTUTestScan(str(root), "scan7", (W, H), n_views=3, full_wh=(W, H))
    xyz0, _ = eval_pipeline.run_scan(model, scan, conf=0.0, min_geo_consistent=0)
    # ground truth built around the fused cloud: a jittered subset of it as the STL
    pts = xyz0.cpu().numpy()
    stl = pts[rng.permutation(len(pts))[: len(pts) // 3]] + rng.normal(0, 0.5, (len(pts) // 3, 3))
    gt = str(tmp_path / "gt")
    synth_dtu.write_ground_truth(gt, 7, stl.astype(np.float32), ground_z=float(np.median(stl[:, 2])))
    ply = str(tmp_path / "points" / "scan7.ply")
    (tmp_path / "points").mkdir()
    xyz, _, scores = eval_pipeline.run_scan(model, scan, conf=0.0, min_geo_consistent=0,
                                            ply_path=ply, dtu_gt=gt)
    direct = dtu_eval.evaluate_scan(xyz, 7, gt)
    from_ply = dtu_eval.evaluate_scan(ply, 7, gt)
    saved = json.loads((tmp_path / "points" / "scan7_scores.json").read_text())
    keys = ("acc", "comp", "overall", "acc_median", "comp_median", "acc_var", "comp_var",
            "n_acc", "n_comp", "n_data", "n_thinned", "n_stl")
    assert scores["n_acc"] > 100 and scores["n_comp"] > 100
    for k in keys:
        assert scores[k] == direct[k] == from_ply[k] == saved[k], k
