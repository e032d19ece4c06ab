"""Tanks and Temples scoring on the GPU against the float64 restatement (oracle/tnt_eval_oracle.py):
crop, voxel means and nearest neighbours bit for bit, an ICP update to 1e-9, seeded scenes end to
end, run-to-run reproducibility and eval_pipeline --tnt_gt on a synthetic COLMAP capture."""
import json
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import ops, synth, synth_scenes, synth_tnt
from casmvsnet_pl_b200 import tnt_eval as E
from oracle import tnt_eval_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cloud(rng, n, scale=3.0):
    return (rng.normal(size=(n, 3)) * scale).astype(np.float32)


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_transform_and_crop_are_bit_identical(axis):
    rng = np.random.default_rng(axis)
    p = _cloud(rng, 300_000)
    # points exactly on polygon vertices, on edges and on the axis bounds
    poly = np.array([[-2.0, -1.0], [2.5, -1.5], [3.0, 2.0], [0.0, 1.0], [-2.5, 2.5]])
    u, v = O.plane_axes(axis)
    extra = np.zeros((len(poly) * 3, 3), np.float32)
    for k, (a, b) in enumerate(poly):
        extra[3 * k, [u, v]] = a, b
        m = (poly[k] + poly[(k + 1) % len(poly)]) / 2
        extra[3 * k + 1, [u, v]] = m
        extra[3 * k + 2, [u, v]] = m
        extra[3 * k + 2, axis] = 1.5
    p = np.concatenate([p, extra])
    T = synth_tnt.similarity(np.random.default_rng(10 + axis), (0.5, 2.0), 1.0)
    vol = (axis, -1.0, 1.5, poly)
    got, idx = ops.tnt_transform_crop(torch.from_numpy(p).to(DEV), T,
                                      (axis, -1.0, 1.5, torch.from_numpy(poly).to(DEV)))
    want_x = O.transform(p, T)
    want_m = O.crop_mask(want_x, *vol)
    assert np.array_equal(idx.cpu().numpy(), np.nonzero(want_m)[0])
    assert np.array_equal(got.cpu().numpy().view(np.uint32), want_x[want_m].view(np.uint32))
    # identity: the crop of the points as they are, including the hand-placed ones
    got2, idx2 = ops.tnt_transform_crop(torch.from_numpy(p).to(DEV), None,
                                        (axis, -1.0, 1.5, torch.from_numpy(poly).to(DEV)))
    assert np.array_equal(idx2.cpu().numpy(), np.nonzero(O.crop_mask(p, *vol))[0])
    xf = ops.tnt_transform_crop(torch.from_numpy(p).to(DEV), T)
    assert np.array_equal(xf.cpu().numpy().view(np.uint32), want_x.view(np.uint32))


@pytest.mark.parametrize("voxel", [0.05, 0.3])
def test_voxel_downsample_is_bit_identical(voxel):
    rng = np.random.default_rng(1)
    p = _cloud(rng, 500_000, 2.0)
    got = E.voxel_downsample(torch.from_numpy(p).to(DEV), voxel).cpu().numpy()
    want = O.voxel_downsample(p, voxel)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_voxel_grid_too_fine_is_refused():
    p = torch.tensor([[0, 0, 0], [1000, 0, 0]], dtype=torch.float32, device=DEV)
    with pytest.raises(ValueError, match="2\\^20"):
        E.voxel_downsample(p, 1e-4)


@pytest.mark.parametrize("case", ["random", "ties"])
def test_nearest_neighbours_are_bit_identical(case):
    rng = np.random.default_rng(2)
    if case == "random":
        t, q = _cloud(rng, 200_000, 1.0), _cloud(rng, 100_000, 1.2)
        cap = 0.05
    else:   # a lattice of step 1/4 and queries at the centres of its cells: 8-way exact ties
        g = np.arange(-20, 20) * 0.25
        t = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
        t = t[rng.permutation(len(t))]
        q = (rng.integers(-20, 19, (50_000, 3)) * 0.25 + 0.125).astype(np.float32)
        cap = 0.3
    lo, hi = np.minimum(t.min(0), q.min(0)), np.maximum(t.max(0), q.max(0))
    grid = E.NNGrid(torch.from_numpy(t).to(DEV), lo, hi, cap, cap / 4)
    d, i = grid.query(torch.from_numpy(q).to(DEV))
    wd, wi = O.nearest(q, t, cap)
    assert np.array_equal(i.cpu().numpy(), wi)
    assert np.array_equal(d.cpu().numpy(), wd)
    if case == "ties":
        assert (wi >= 0).all()


def test_one_icp_iteration_matches_to_1e9():
    rng = np.random.default_rng(3)
    t = _cloud(rng, 100_000, 1.0)
    s = (t[:80_000] @ np.array([[0.99, -0.1, 0], [0.1, 0.99, 0], [0, 0, 1]], np.float32).T * 1.05
         + 0.01).astype(np.float32)
    T = synth_tnt.similarity(np.random.default_rng(4), (0.98, 1.02), 0.01)
    T[:3, :3] = np.eye(3) * 1.001
    origin = np.array([0.1, -0.2, 0.3])
    td = torch.from_numpy(t).to(DEV)
    grid = E.NNGrid(td, t.min(0), t.max(0), 0.1, 0.02)
    q = ops.tnt_transform_crop(torch.from_numpy(s).to(DEV), T)
    d, idx = grid.query(q)
    mom = ops.tnt_icp_moments(q, td, idx, origin)
    got = E.icp_update(mom, origin)
    qo = O.transform(s, T)
    wd, wi = O.nearest(qo, t, 0.1)
    assert np.array_equal(idx.cpu().numpy(), wi)
    sel = wi >= 0
    want = O.umeyama(qo[sel], t[wi[sel]])
    assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max()
    m = mom.cpu().numpy()
    assert m[0] == sel.sum()
    assert abs(m[1] - (wd[sel] ** 2).sum()) <= 1e-9 * m[1]
    # the moment reduction is the same bits on every call
    assert torch.equal(mom, ops.tnt_icp_moments(q, td, idx, origin))


def _scene(tmp_path, seed):
    return synth_tnt.make_scene(str(tmp_path / f"s{seed}"), n_gt=120_000, n_rec=100_000, seed=seed)


def _agree(n_got, n_want, d, tau):
    """counts may differ only by the points whose distance lies within 1e-9 of tau"""
    return abs(n_got - n_want) <= int((np.abs(np.asarray(d) - tau) <= 1e-9).sum())


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_seeded_scene_end_to_end_matches_the_oracle(tmp_path, seed):
    s = _scene(tmp_path, seed)
    r = E.evaluate_scene(s["ply"], s["run_dir"], s["gt_dir"], s["scene"], tau=s["tau"], seed=seed,
                         images=s["images"], return_arrays=True)
    tau = s["tau"]
    assert r["alignment"]["inliers"] == r["alignment"]["pairs"] - 3     # the perturbed cameras
    rec = E.read_points(s["ply"])
    gt = E.read_points(os.path.join(s["gt_dir"], s["scene"], f"{s['scene']}.ply"))
    vol = E.read_crop(os.path.join(s["gt_dir"], s["scene"], f"{s['scene']}.json"))
    T = np.array(r["T"])
    true = rec.astype(np.float64) @ s["rec_to_gt"][:3, :3].T + s["rec_to_gt"][:3, 3]
    inside = O.crop_mask(true.astype(np.float32), *vol)
    got = rec[inside].astype(np.float64) @ T[:3, :3].T + T[:3, 3]
    err = np.linalg.norm(got - true[inside], axis=1)
    assert err.max() < 0.2 * tau, err.max()
    want = O.evaluate(rec, gt, np.array(r["alignment"]["T0"]), vol, tau)
    for k, st in enumerate(want["stages"]):
        assert r["stages"][k]["iterations"] == st[1]
        assert np.abs(np.array(r["stages"][k]["T"]) - st[0]).max() < 1e-6
    n1 = int((r["d1"] < tau).sum().item())
    n2 = int((r["d2"] < tau).sum().item())
    assert r["counts"]["score_source"] == want["n_source"]
    assert r["counts"]["score_target"] == want["n_target"]
    assert _agree(n1, int((want["d1"] < tau).sum()), want["d1"], tau)
    assert _agree(n2, int((want["d2"] < tau).sum()), want["d2"], tau)
    for k in ("precision", "recall", "fscore"):
        assert abs(r[k] - want[k]) <= 2.0 / min(want["n_source"], want["n_target"]), k
    assert 0.5 < r["fscore"] <= 1.0


def test_two_runs_give_identical_json(tmp_path):
    s = _scene(tmp_path, 5)
    outs = []
    for k in range(2):
        r = E.evaluate_scene(s["ply"], s["run_dir"], s["gt_dir"], s["scene"], tau=s["tau"],
                             images=s["images"])
        path = tmp_path / f"r{k}.json"
        E.write_json(str(path), r)
        d = json.loads(path.read_text())
        d.pop("time_s")
        outs.append(d)
    assert outs[0] == outs[1]
    assert len(outs[0]["curve_precision"]) == 499 and len(outs[0]["stages"]) == 3


def test_cli_writes_scores(tmp_path):
    s = _scene(tmp_path, 6)
    out = tmp_path / "scores.json"
    E.main(["--ply", s["ply"], "--run_dir", s["run_dir"], "--gt_dir", s["gt_dir"], "--scene",
            s["scene"], "--tau", str(s["tau"]), "--images", s["images"], "--out", str(out)])
    d = json.loads(out.read_text())
    assert set(d) >= {"precision", "recall", "fscore", "tau", "alignment", "stages", "counts",
                      "curve_precision", "curve_recall", "time_s"}


def _tree_bytes(d):
    return {os.path.relpath(os.path.join(r, n), d): open(os.path.join(r, n), "rb").read()
            for r, _, files in os.walk(d) for n in files}


def test_eval_pipeline_tnt_gt_end_to_end(tmp_path):
    root = tmp_path / "Barn"                                # a training scene's name: tau 0.01
    synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), n_points=3000, seed=7)
    gt = tmp_path / "gt"
    synth_tnt.write_gt_for_colmap(str(root), str(gt), "Barn", n_points=100_000)
    torch.manual_seed(0)
    from casmvsnet_pl_b200 import ABN
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    model = CascadeMVSNet(norm_act=ABN)
    synth.randomize_model_(model, 0)
    ckpt = tmp_path / "weights.pt"
    torch.save(model.state_dict(), ckpt)
    common = ["--dataset_name", "colmap", "--root_dir", str(root), "--img_wh", "128", "96",
              "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0", "--ckpt", str(ckpt)]
    ep.main(common + ["--out", str(tmp_path / "plain")])
    ep.main(common + ["--out", str(tmp_path / "tnt"), "--tnt_gt", str(gt)])
    plain, tnt = _tree_bytes(tmp_path / "plain"), _tree_bytes(tmp_path / "tnt")
    key = os.path.join("points", "Barn_tnt.json")
    assert {k: v for k, v in tnt.items() if k != key} == plain       # nothing else changes
    got = json.loads(tnt[key])
    assert got["counts"]["source"] > 0
    again = E.evaluate_scene(str(tmp_path / "tnt" / "points" / "Barn.ply"),
                             str(tmp_path / "tnt" / "Barn"), str(gt), "Barn")
    got.pop("time_s")
    again = json.loads(json.dumps({k: v for k, v in again.items() if k != "time_s"}))
    assert got == again
