"""Statistical outlier removal on the GPU (cloud_filter.py, csrc/pcd_eval.cu): the mean neighbour
distances, the statistics and the mask bit for bit against the float64 oracle
(oracle/cloud_filter_oracle.py) on a noisy sphere with outliers, a lattice with duplicates, a tiny
cluster with far points and a cloud of k + 1 points; reproducibility, permutation, the refusals,
the command line, and eval_pipeline --remove_outliers end to end."""
import json
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, cloud_filter, io, synth, synth_dtu, synth_scenes, synth_tnt
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import cloud_filter_oracle as O
from test_cloud_filter import noisy_sphere

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _sphere():
    return noisy_sphere(198_000, 2_000, 5)


def _lattice():
    rng = np.random.default_rng(1)
    g = np.arange(30, dtype=np.float32)
    p = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    return np.concatenate([p, p[rng.choice(len(p), 3000, replace=False)]])[rng.permutation(len(p) + 3000)]


def _cluster():
    rng = np.random.default_rng(2)
    far = rng.normal(size=(100, 3))
    far *= 1e3 / np.linalg.norm(far, axis=1, keepdims=True)
    return np.concatenate([rng.uniform(0, 1e-3, (100_000, 3)), far]).astype(np.float32)


CLOUDS = {"sphere": _sphere, "lattice": _lattice, "cluster": _cluster}
_cache = {}


def _cloud(name):
    if name not in _cache:
        _cache[name] = CLOUDS[name]()
    return _cache[name]


@pytest.mark.parametrize("k", [1, 20, 64])
@pytest.mark.parametrize("name", list(CLOUDS) + ["k_plus_1"])
def test_mean_distance_statistics_and_mask_are_bit_identical_to_the_oracle(name, k):
    xyz = (np.random.default_rng(k).normal(size=(k + 1, 3)).astype(np.float32)
           if name == "k_plus_1" else _cloud(name))
    m = cloud_filter.mean_neighbour_distance(_cuda(xyz), k).cpu().numpy()
    want = O.mean_distance(xyz, k)
    assert np.array_equal(m, want), f"{int((m != want).sum())} of {len(m)} differ"
    keep, st = cloud_filter.remove_statistical_outliers(_cuda(xyz), k, 2.0)
    keep_o, _, mu, sigma, thr = O.remove_statistical_outliers(xyz, k, 2.0)
    assert (st["mean"], st["std"], st["threshold"]) == (mu, sigma, thr)
    assert np.array_equal(keep.cpu().numpy(), keep_o)
    assert st["points"] == len(xyz) and st["kept"] == int(keep_o.sum()) and st["k"] == k
    assert set(st["time_s"]) == {"bounds_keys_s", "sort_cells_s", "search_s", "statistics_s"}


def test_chunk_sums_and_a_ratio_sweep_match_the_oracle():
    xyz = _cloud("sphere")
    m = cloud_filter.mean_neighbour_distance(_cuda(xyz), 20)
    for r in (0.5, 1.0, 3.0):
        st, mask, counts, chunks = cloud_filter.ops.pcd_sor_keep(m, r)
        mu, sigma, thr, chunks_o = O.statistics(m.cpu().numpy(), r)
        assert st.tolist() == [mu, sigma, thr]
        assert np.array_equal(chunks.cpu().numpy(), chunks_o)
        assert np.array_equal(mask.cpu().numpy().astype(bool), m.cpu().numpy() <= thr)
        assert int(counts.sum()) == int(mask.sum())


def test_outliers_go_and_two_runs_agree():
    xyz = _cuda(_cloud("sphere"))
    k1, s1 = cloud_filter.remove_statistical_outliers(xyz)
    k2, s2 = cloud_filter.remove_statistical_outliers(xyz)
    assert torch.equal(k1, k2)
    assert {k: v for k, v in s1.items() if k != "time_s"} == {k: v for k, v in s2.items() if k != "time_s"}
    assert not k1[198_000:].any() and k1[:198_000].float().mean() > 0.97
    m1 = cloud_filter.mean_neighbour_distance(xyz, 20)
    m2 = cloud_filter.mean_neighbour_distance(xyz, 20)
    assert torch.equal(m1, m2)
    pts, idx, st = cloud_filter.filter_points(xyz)
    assert torch.equal(idx, k1.nonzero().squeeze(1)) and torch.equal(pts, xyz[k1])
    assert st["kept"] == len(idx)


@pytest.mark.parametrize("name", ["sphere", "lattice"])
def test_permuting_the_input_permutes_the_distances(name):
    xyz = _cloud(name)
    perm = np.random.default_rng(9).permutation(len(xyz))
    m = cloud_filter.mean_neighbour_distance(_cuda(xyz), 20).cpu().numpy()
    mp = cloud_filter.mean_neighbour_distance(_cuda(xyz[perm]), 20).cpu().numpy()
    assert np.array_equal(mp, m[perm])


def test_refusals_name_their_values():
    xyz = _cuda(_cloud("lattice"))
    n = len(xyz)
    need = n * cloud_filter.BYTES_PER_POINT
    with pytest.raises(_lib.CasMVSError, match=f"filtering {n} points needs {need} bytes .* but "
                                               f"1000 bytes are available"):
        cloud_filter.remove_statistical_outliers(xyz, max_bytes=1000)
    cloud_filter.remove_statistical_outliers(xyz, max_bytes=need)
    bad = xyz.clone()
    bad[17, 2] = float("nan")
    with pytest.raises(ValueError, match="non-finite coordinate at point 17"):
        cloud_filter.remove_statistical_outliers(bad)
    with pytest.raises(ValueError, match="a cloud of 20 points cannot be filtered with k = 20"):
        cloud_filter.remove_statistical_outliers(xyz[:20])
    with pytest.raises(ValueError, match="got torch.float64 on cuda"):
        cloud_filter.remove_statistical_outliers(xyz.double())
    with pytest.raises(ValueError, match="k must be an integer in 1..64, got 65"):
        cloud_filter.remove_statistical_outliers(xyz, k=65)


def test_cli_keeps_every_property_of_the_kept_points(tmp_path, capsys):
    xyz = _cloud("sphere")[::4]
    v = np.zeros(len(xyz), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"),
                                  ("ny", "<f4"), ("nz", "<f4"), ("red", "u1"), ("green", "u1"),
                                  ("blue", "u1")])
    v["x"], v["y"], v["z"] = xyz.T
    n = xyz / np.linalg.norm(xyz, axis=1, keepdims=True)
    v["nx"], v["ny"], v["nz"] = n.T
    v["red"] = np.arange(len(v)) % 256
    cloud_filter.write_vertices(tmp_path / "in.ply", v)
    st = cloud_filter.main(["--ply", str(tmp_path / "in.ply"), "--out", str(tmp_path / "out.ply"),
                            "--neighbours", "12", "--std_ratio", "1.5"])
    assert "kept" in capsys.readouterr().out
    keep, _ = cloud_filter.remove_statistical_outliers(_cuda(xyz), 12, 1.5)
    keep = keep.cpu().numpy()
    assert st["kept"] == keep.sum() < len(v)
    cloud_filter.write_vertices(tmp_path / "want.ply", v[keep])
    assert (tmp_path / "out.ply").read_bytes() == (tmp_path / "want.ply").read_bytes()
    out = io.read_ply(tmp_path / "out.ply")
    assert out.dtype.names == v.dtype.names and np.array_equal(out["nx"], v["nx"][keep])


# ------------------------------------------------------------------------------ eval_pipeline
def _model_ckpt(tmp_path):
    from casmvsnet_pl_b200 import ABN
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN)
    synth.randomize_model_(model, 0)
    ckpt = tmp_path / "weights.pt"
    torch.save(model.state_dict(), ckpt)
    return model, ckpt


def _tree(d):
    return {os.path.relpath(os.path.join(r, n), d): open(os.path.join(r, n), "rb").read()
            for r, _, files in os.walk(d) for n in files}


def test_eval_pipeline_filters_the_written_and_scored_cloud_tnt(tmp_path, capsys):
    root = tmp_path / "Barn"
    synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), n_points=3000, seed=7)
    gt = tmp_path / "gt"
    synth_tnt.write_gt_for_colmap(str(root), str(gt), "Barn", n_points=100_000)
    _, ckpt = _model_ckpt(tmp_path)
    common = ["--dataset_name", "colmap", "--root_dir", str(root), "--img_wh", "128", "96",
              "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0", "--ckpt", str(ckpt),
              "--tnt_gt", str(gt), "--tnt_tau", "0.04"]
    ep.main(common + ["--out", str(tmp_path / "plain")])
    capsys.readouterr()
    ep.main(common + ["--out", str(tmp_path / "f"), "--remove_outliers", "--outlier_neighbours",
                      "10", "--outlier_std", "1.0"])
    log = capsys.readouterr().out
    assert sum("removed outliers" in ln for ln in log.splitlines()) == 1
    plain, filt = _tree(tmp_path / "plain"), _tree(tmp_path / "f")
    ply = os.path.join("points", "Barn.ply")
    cloud_filter.main(["--ply", str(tmp_path / "plain" / ply), "--out", str(tmp_path / "cli.ply"),
                       "--neighbours", "10", "--std_ratio", "1.0"])
    assert (tmp_path / "cli.ply").read_bytes() == filt[ply]
    assert len(filt[ply]) < len(plain[ply])
    changed = {ply, os.path.join("points", "Barn_tnt.json")}
    assert {k: v for k, v in filt.items() if k not in changed} == \
        {k: v for k, v in plain.items() if k not in changed}
    pts = io.read_ply(tmp_path / "cli.ply")
    xyz = _cuda(np.stack([pts["x"], pts["y"], pts["z"]], 1))
    from casmvsnet_pl_b200 import tnt_eval
    again = tnt_eval.evaluate_scene(xyz, str(tmp_path / "f" / "Barn"), str(gt), "Barn", tau=0.04)
    saved = json.loads(filt[os.path.join("points", "Barn_tnt.json")])
    for key in ("precision", "recall", "fscore"):
        assert saved[key] == again[key]


@pytest.mark.parametrize("skip", [1, 2])
def test_eval_pipeline_poisson_meshes_the_filtered_points(tmp_path, capsys, skip):
    root = tmp_path / "capture"
    synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), n_points=3000, seed=7)
    _, ckpt = _model_ckpt(tmp_path)
    common = ["--dataset_name", "colmap", "--root_dir", str(root), "--img_wh", "128", "96",
              "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0", "--ckpt", str(ckpt),
              "--skip", str(skip), "--mesh", "--mesh_method", "poisson", "--poisson_depth", "7"]
    ep.main(common + ["--out", str(tmp_path / "plain")])
    capsys.readouterr()
    ep.main(common + ["--out", str(tmp_path / "f"), "--remove_outliers", "--outlier_std", "1.0"])
    log = [ln for ln in capsys.readouterr().out.splitlines() if "removed outliers" in ln]
    assert len(log) == (1 if skip == 1 else 2)
    assert any("(poisson points)" in ln for ln in log) == (skip != 1)
    plain, filt = _tree(tmp_path / "plain"), _tree(tmp_path / "f")
    mesh_file = os.path.join("mesh", "capture.ply")
    assert mesh_file in filt and filt[mesh_file] != plain[mesh_file]


def test_eval_pipeline_poisson_points_are_the_filtered_cloud(tmp_path, monkeypatch):
    """With --skip 1 Poisson receives exactly the points and colours the PLY holds."""
    from casmvsnet_pl_b200 import poisson
    root = tmp_path / "capture"
    synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), n_points=3000, seed=7)
    _, ckpt = _model_ckpt(tmp_path)
    seen = {}
    real = poisson.poisson_mesh

    def spy(pts, cols, **kw):
        seen["pts"], seen["cols"] = pts.cpu().numpy(), cols.cpu().numpy()
        return real(pts, cols, **kw)
    monkeypatch.setattr(poisson, "poisson_mesh", spy)
    ep.main(["--dataset_name", "colmap", "--root_dir", str(root), "--img_wh", "128", "96",
             "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0", "--ckpt", str(ckpt),
             "--mesh", "--mesh_method", "poisson", "--poisson_depth", "7", "--remove_outliers",
             "--out", str(tmp_path / "f")])
    v = io.read_ply(tmp_path / "f" / "points" / "capture.ply")
    assert np.array_equal(seen["pts"], np.stack([v["x"], v["y"], v["z"]], 1))
    assert np.array_equal(seen["cols"], np.stack([v["red"], v["green"], v["blue"]], 1))


def test_run_scan_scores_the_filtered_cloud_dtu(tmp_path):
    from casmvsnet_pl_b200 import dtu_eval
    root = tmp_path / "scan7"
    synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), n_points=3000, seed=7)
    model, _ = _model_ckpt(tmp_path)
    model = model.eval().cuda()
    scan = ep.ColmapScan(str(root), None, (128, 96), 3, 192.0)
    xyz0, _ = ep.run_scan(model, scan, conf=0.0, min_geo_consistent=0)
    rng = np.random.default_rng(0)
    pts = xyz0.cpu().numpy()
    stl = pts[rng.permutation(len(pts))[: len(pts) // 3]] + rng.normal(0, 0.01, (len(pts) // 3, 3))
    gt = str(tmp_path / "gt")
    synth_dtu.write_ground_truth(gt, 7, stl.astype(np.float32), ground_z=float(np.median(stl[:, 2])),
                                 res=0.05)
    logs = []
    xyz, rgb, scores = ep.run_scan(model, scan, conf=0.0, min_geo_consistent=0, dtu_gt=gt,
                                   ply_path=str(tmp_path / "scan7.ply"), log=logs.append,
                                   outlier_filter=dict(k=8))
    kept, idx, st = cloud_filter.filter_points(xyz0, 8)
    assert torch.equal(xyz, kept) and len(xyz) < len(xyz0)
    assert any("removed outliers" in m and f"kept {len(xyz)} of {len(xyz0)}" in m for m in logs)
    again = dtu_eval.evaluate_scan(kept, 7, gt)
    assert {k: v for k, v in scores.items() if k != "time_s"} == \
        {k: v for k, v in again.items() if k != "time_s"}
    v = io.read_ply(tmp_path / "scan7.ply")
    assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], 1), kept.cpu().numpy())
    assert np.array_equal(np.stack([v["red"], v["green"], v["blue"]], 1), rgb.cpu().numpy())


def test_run_scan_writes_a_tiny_cloud_unfiltered(tmp_path):
    root = tmp_path / "capture"
    synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), n_points=3000, seed=7)
    model, _ = _model_ckpt(tmp_path)
    model = model.eval().cuda()
    scan = ep.ColmapScan(str(root), None, (128, 96), 3, 192.0)
    xyz0, rgb0 = ep.run_scan(model, scan, conf=0.0, min_geo_consistent=0, skip=100_000)
    logs = []
    xyz, rgb = ep.run_scan(model, scan, conf=0.0, min_geo_consistent=0, skip=100_000,
                           log=logs.append, outlier_filter=dict(k=64))
    assert len(xyz0) <= 64 and torch.equal(xyz, xyz0) and torch.equal(rgb, rgb0)
    assert any("outliers not removed" in m for m in logs)
