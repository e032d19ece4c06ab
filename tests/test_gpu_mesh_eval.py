"""Mesh scoring on the GPU (mesh_sample.py, csrc/mesh_sample.cu, dtu_eval.evaluate_mesh,
tnt_eval.evaluate_mesh, eval_pipeline --mesh_score): surface samples bit for bit against the
numpy restatement (oracle/mesh_sample_oracle.py) on four meshes, byte reproducibility, agreement
with the point scorers on the oracle's samples, analytic DTU and Tanks and Temples checks, the
error clouds, eval_pipeline end to end and the refusals."""
import json
import math
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import (_lib, dtu_eval, io, mesh, mesh_sample, simplify, synth, synth_dtu,
                               synth_scenes, synth_tnt, tnt_eval)
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import mesh_sample_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


_CACHE = {}


def _sphere_mesh():
    if "sphere" not in _CACHE:
        views = synth_scenes.sphere_scene(12, (240, 180), seed=3, device=DEV)
        v, _, f, _ = mesh.mesh_views([x["points"] for x in views], [x["depth"] for x in views],
                                     [x["image"] for x in views], [x["P"] for x in views], voxel=0.05)
        _CACHE["sphere"] = (v.cpu().numpy(), f.cpu().numpy())
    return _CACHE["sphere"]


def _decimated():
    v, f = _sphere_mesh()
    V, _, F, _ = simplify.simplify_mesh(_cuda(v), torch.zeros(len(v), 3, dtype=torch.uint8, device=DEV),
                                        _cuda(f), max(1, len(f) // 20))
    return V.cpu().numpy(), F.cpu().numpy()


def _degenerate():
    v = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0], [7, 7, 7], [0.5, 0.5, 0.25],
                    [-1e-3, 3, 1]])
    f = np.int32([[0, 1, 2], [0, 0, 1], [2, 2, 2], [0, 1, 3], [5, 2, 6], [1, 5, 0], [3, 3, 6]])
    return v, f                                  # repeats, a point, collinear, vertex 4 unused


def _sliver():
    v = np.float32([[0, 0, 0], [1500, 0, 0], [1500, 1e-3, 2e-3], [0, 1, 0], [1, 1, 0]])
    f = np.int32([[3, 0, 4], [0, 1, 2], [4, 3, 0]])
    return v, f


MESHES = {"sphere_tsdf": (_sphere_mesh, 0.01), "sphere_decimated": (_decimated, 0.01),
          "degenerate": (_degenerate, 0.07), "sliver": (_sliver, 1.0)}


@pytest.mark.parametrize("name", list(MESHES))
def test_samples_are_bit_identical_to_the_oracle(name):
    make, s = MESHES[name]
    v, f = make()
    want, n_w, cnt_w, off_w = O.sample(v, f, s)
    V, F = _cuda(v), _cuda(f).int()
    n, cnt, start = mesh_sample.sample_counts(V, F, s)
    assert np.array_equal(n.cpu().numpy(), n_w) and np.array_equal(cnt.cpu().numpy(), cnt_w)
    assert np.array_equal(start.cpu().numpy(), off_w)
    got = mesh_sample.sample_surface(V, F, s).cpu().numpy()
    assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    if name == "sliver":
        assert cnt_w[1] >= 1_000_000
    if name.startswith("sphere"):
        assert len(got) > 100_000


def test_two_runs_give_the_same_bytes():
    v, f = _sphere_mesh()
    a = mesh_sample.sample_surface(_cuda(v), _cuda(f), 0.01).cpu().numpy().tobytes()
    b = mesh_sample.sample_surface(_cuda(v), _cuda(f).long(), 0.01).cpu().numpy().tobytes()
    assert a == b


def _drop_time(r):
    return {k: v for k, v in r.items() if k != "time_s"}


def _same(a, b):
    """Equality of score dicts, NaN equal to NaN."""
    assert set(a) == set(b)
    for k in a:
        x, y = a[k], b[k]
        if torch.is_tensor(x):
            assert torch.equal(x, y), k
        elif isinstance(x, float) and math.isnan(x):
            assert isinstance(y, float) and math.isnan(y), k
        else:
            assert x == y, k


# ------------------------------------------------------------------------------ DTU
def _height_bounds(L):
    """(max slope |grad z|, bound on the Hessian's norm) of synth_dtu._height, from its closed
    form: grad and second derivatives of 0.08 L sin(2 pi x/L) cos(2 pi y/L) + 0.05 L cos(pi x/L)."""
    w, a, b = 2 * np.pi / L, 0.08 * L, 0.05 * L
    g = math.hypot(a * w + b * np.pi / L, a * w)
    hess = 2 * a * w * w + b * (np.pi / L) ** 2          # |f_xx| + |f_xy| bound per row
    return g, hess


def test_dtu_mesh_scores_equal_the_point_scores_of_the_oracle_samples(tmp_path):
    gt = str(tmp_path / "gt")
    synth_dtu.make_scene(gt, scan=3, n_stl=40_000, n_data=1000, seed=2)
    stl = dtu_eval.read_points(dtu_eval.stl_path(gt, 3))
    v, f, _, _ = synth_dtu.height_mesh(stl, 0.6)
    got = dtu_eval.evaluate_mesh((_cuda(v), _cuda(f)), 3, gt, return_arrays=True)
    want = dtu_eval.evaluate_scan(_cuda(O.sample(v, f, dtu_eval.DST)[0]), 3, gt, return_arrays=True)
    assert got["n_faces"] == len(f) and got["n_samples"] == want["n_data"] and got["spacing"] == 0.2
    assert got["time_s"]["sample_s"] >= 0
    samples = got.pop("samples")
    assert len(samples) == got["n_samples"]
    for k in ("n_faces", "n_samples", "spacing"):
        got.pop(k)
    _same(_drop_time(got), _drop_time(want))


def test_dtu_analytic_surface(tmp_path):
    from scipy.spatial import cKDTree
    gt = str(tmp_path / "gt")
    synth_dtu.make_scene(gt, scan=1, n_stl=100_000, n_data=1000, seed=0)
    stl = dtu_eval.read_points(dtu_eval.stl_path(gt, 1))
    v, f, L, diag = synth_dtu.height_mesh(stl, 0.5)
    g, hess = _height_bounds(L)
    chord = hess * diag * diag / 2                   # linear interpolation error over a triangle
    # the mean distance from the true surface to the nearest STL point (~0.1 mm at 25 / mm^2),
    # per unit of surface area as the samples are spread
    rng = np.random.default_rng(5)
    xy = rng.uniform(stl[:, :2].min(0), stl[:, :2].max(0), (200_000, 2)) - synth_dtu.CENTER[:2]
    z = synth_dtu._height(xy[:, 0], xy[:, 1], L)
    e = 1e-4
    zx = (synth_dtu._height(xy[:, 0] + e, xy[:, 1], L) - synth_dtu._height(xy[:, 0] - e, xy[:, 1], L)) / (2 * e)
    zy = (synth_dtu._height(xy[:, 0], xy[:, 1] + e, L) - synth_dtu._height(xy[:, 0], xy[:, 1] - e, L)) / (2 * e)
    area = np.sqrt(1 + zx * zx + zy * zy)
    assert np.hypot(zx, zy).max() <= g
    q = np.c_[xy, z] + synth_dtu.CENTER
    d = cKDTree(stl.astype(np.float64)).query(q)[0]
    mean_nn = float((d * area).sum() / area.sum())
    assert 0.08 < mean_nn < 0.13
    r = dtu_eval.evaluate_mesh((_cuda(v), _cuda(f)), 1, gt)
    assert r["n_acc"] > 30_000 and r["n_comp"] > 30_000
    assert r["acc"] <= 1.05 * mean_nn + chord, (r["acc"], mean_nn, chord)
    # an STL point is within chord of the mesh, and every sample within dst of a kept one
    assert r["comp"] <= chord + dtu_eval.DST + dtu_eval.DST / math.sqrt(3), r["comp"]
    delta = 1.0
    v2, _, _, _ = synth_dtu.height_mesh(stl, 0.5, shift=delta)
    s = dtu_eval.evaluate_mesh((_cuda(v2), _cuda(f)), 1, gt)
    lo = (delta - chord) / math.sqrt(1 + g * g)      # delta . min cos(slope), less the chord
    assert lo <= s["acc"] <= delta + 1.05 * mean_nn + chord, (s["acc"], lo)


def test_error_clouds_and_the_command_line(tmp_path):
    gt = str(tmp_path / "gt")
    synth_dtu.make_scene(gt, scan=2, n_stl=30_000, n_data=1000, seed=4)
    stl = dtu_eval.read_points(dtu_eval.stl_path(gt, 2))
    v, f, _, _ = synth_dtu.height_mesh(stl, 0.7)
    mdir = tmp_path / "mesh"
    mdir.mkdir()
    mesh.write_mesh_ply(mdir / "scan2.ply", v, np.zeros((len(v), 3), np.uint8), f)
    outs = []
    for k in range(2):
        e = tmp_path / f"err{k}"
        dtu_eval.main(["--mesh_dir", str(mdir), "--gt_dir", gt, "--scans", "2", "--error_dir", str(e),
                       "--out", str(tmp_path / f"s{k}.json")])
        outs.append({n: (e / n).read_bytes() for n in ("scan2_data2stl.ply", "scan2_stl2data.ply")})
    assert outs[0] == outs[1]
    saved = json.loads((tmp_path / "s0.json").read_text())["scans"][0]
    r = dtu_eval.evaluate_mesh(str(mdir / "scan2.ply"), 2, gt, return_arrays=True)
    assert _drop_time(saved) == json.loads(json.dumps(_drop_time(
        {k: x for k, x in r.items() if not torch.is_tensor(x)})))
    d2s = io.read_ply(tmp_path / "err0" / "scan2_data2stl.ply")
    s2d = io.read_ply(tmp_path / "err0" / "scan2_stl2data.ply")
    assert len(d2s) == r["n_thinned"] and len(s2d) == r["n_stl"]
    data = r["samples"][r["kept"]].cpu().numpy()
    assert np.array_equal(np.c_[d2s["x"], d2s["y"], d2s["z"]], data)
    assert np.array_equal(np.c_[s2d["x"], s2d["y"], s2d["z"]], stl)
    for cloud, d, flag in ((d2s, r["Ddata"], r["data_in_mask"]), (s2d, r["Dstl"], r["stl_above_plane"])):
        want = dtu_eval.error_colours(d.cpu().numpy(), flag.cpu().numpy())
        assert np.array_equal(np.c_[cloud["red"], cloud["green"], cloud["blue"]], want)
    # a cloud gets its error clouds too
    pdir = tmp_path / "points"
    pdir.mkdir()
    from casmvsnet_pl_b200.fusion import write_ply
    write_ply(pdir / "scan2.ply", data, np.zeros((len(data), 3), np.uint8))
    dtu_eval.main(["--ply_dir", str(pdir), "--gt_dir", gt, "--scans", "2", "--error_dir",
                   str(tmp_path / "errp")])
    assert len(io.read_ply(tmp_path / "errp" / "scan2_data2stl.ply")) > 0


# ------------------------------------------------------------------------------ Tanks and Temples
def _tnt_mesh(sc):
    P, f = synth_tnt.surface_mesh()
    T = np.linalg.inv(sc["rec_to_gt"])
    return (P @ T[:3, :3].T + T[:3, 3]).astype(np.float32), f


def test_tnt_mesh_scores_equal_the_point_scores_of_the_oracle_samples(tmp_path):
    sc = synth_tnt.make_scene(str(tmp_path), n_gt=100_000, n_rec=100_000, seed=1)
    v, f = _tnt_mesh(sc)
    args = (sc["run_dir"], sc["gt_dir"], sc["scene"])
    got = tnt_eval.evaluate_mesh((_cuda(v), _cuda(f)), *args, tau=sc["tau"], images=sc["images"])
    want = tnt_eval.evaluate_scene(_cuda(O.sample(v, f, sc["tau"] / 4)[0]), *args, tau=sc["tau"],
                                   images=sc["images"])
    assert got.pop("n_faces") == len(f) and got.pop("spacing") == sc["tau"] / 4
    assert got.pop("n_samples") == want["counts"]["source"]
    _same(_drop_time(got), _drop_time(want))


def test_tnt_analytic_surfaces_score_at_least_the_noisy_cloud(tmp_path):
    sc = synth_tnt.make_scene(str(tmp_path), seed=0)
    v, f = _tnt_mesh(sc)
    args = (sc["run_dir"], sc["gt_dir"], sc["scene"])
    m = tnt_eval.evaluate_mesh((_cuda(v), _cuda(f)), *args, tau=sc["tau"], images=sc["images"])
    p = tnt_eval.evaluate_scene(sc["ply"], *args, tau=sc["tau"], images=sc["images"])
    assert m["precision"] >= 0.99, m["precision"]
    assert m["fscore"] >= p["fscore"], (m["fscore"], p["fscore"])
    ply = tmp_path / "mesh.ply"
    mesh.write_mesh_ply(ply, v, np.zeros((len(v), 3), np.uint8), f)
    out = tmp_path / "m.json"
    tnt_eval.main(["--mesh", str(ply), "--run_dir", sc["run_dir"], "--gt_dir", sc["gt_dir"],
                   "--scene", sc["scene"], "--tau", str(sc["tau"]), "--images", sc["images"],
                   "--out", str(out)])
    saved = json.loads(out.read_text())
    assert saved["fscore"] == m["fscore"] and saved["n_samples"] == m["n_samples"]


# ------------------------------------------------------------------------------ eval_pipeline
def _tree(d):
    """Every file's bytes; a score JSON's parsed content less its timings."""
    out = {}
    for r, _, files in os.walk(d):
        for n in files:
            p = os.path.join(r, n)
            out[os.path.relpath(p, d)] = (_drop_time(json.loads(open(p).read())) if n.endswith(".json")
                                          else open(p, "rb").read())
    return out


def test_eval_pipeline_mesh_score_dtu_route(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from casmvsnet_pl_b200 import ABN
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    root = tmp_path / "dtu"
    (root / "Cameras").mkdir(parents=True)
    (root / "Rectified" / "scan7").mkdir(parents=True)
    rng = np.random.default_rng(0)
    W, H, n = 160, 128, 4
    K4 = synth.intrinsics(0, W, H)
    for vid in range(n):                         # a tenth of the DTU scale: a small mesh area
        t = np.deg2rad(3.0 * vid)
        E = np.eye(4)
        E[:3, :3] = [[np.cos(t), 0, np.sin(t)], [0, 1, 0], [-np.sin(t), 0, np.cos(t)]]
        E[:3, 3] = [-68 * np.sin(t), 0, 68 * (1 - np.cos(t))]
        rows = ["extrinsic"] + [" ".join(f"{v:.6f}" for v in r) for r in E] + ["", "intrinsic"]
        rows += [" ".join(f"{v:.6f}" for v in r) for r in K4] + ["", "42.5 0.265"]
        (root / "Cameras" / f"{vid:08d}_cam.txt").write_text("\n".join(rows) + "\n")
        cv2.imwrite(str(root / "Rectified" / "scan7" / f"rect_{vid + 1:03d}_3_r5000.png"),
                    rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
    (root / "Cameras" / "pair.txt").write_text(
        "4\n0\n3 1 9.0 2 8.0 3 7.0\n1\n3 0 9.0 2 8.0 3 7.0\n2\n3 1 9.0 3 8.0 0 7.0\n3\n3 2 9.0 1 8.0 0 7.0\n")
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN, precision="tf32")
    synth.randomize_model_(model, 0)
    model = model.eval().cuda()
    scan = ep.DTUTestScan(str(root), "scan7", (W, H), n_views=3, full_wh=(W, H))
    xyz0, _ = ep.run_scan(model, scan, conf=0.0, min_geo_consistent=0)
    pts = xyz0.cpu().numpy()
    stl = pts[rng.permutation(len(pts))[: len(pts) // 3]] + rng.normal(0, 0.05, (len(pts) // 3, 3))
    gt = str(tmp_path / "gt")
    synth_dtu.write_ground_truth(gt, 7, stl.astype(np.float32), ground_z=float(np.median(stl[:, 2])))
    outs = {}
    for tag, flag in (("plain", False), ("scored", True)):
        d = tmp_path / tag
        (d / "points").mkdir(parents=True)
        (d / "mesh").mkdir()
        outs[tag] = ep.run_scan(model, scan, conf=0.0, min_geo_consistent=0, dtu_gt=gt,
                                ply_path=str(d / "points" / "scan7.ply"),
                                mesh_path=str(d / "mesh" / "scan7.ply"), mesh_faces=3000,
                                mesh_score=flag)
    assert len(outs["plain"]) == 3 and len(outs["scored"]) == 4
    plain, scored = _tree(tmp_path / "plain"), _tree(tmp_path / "scored")
    key = os.path.join("mesh", "scan7_scores.json")
    assert os.path.join("points", "scan7_scores.json") in plain
    assert {k: v for k, v in scored.items() if k != key} == plain
    saved = json.loads((tmp_path / "scored" / key).read_text())
    again = dtu_eval.evaluate_mesh(str(tmp_path / "scored" / "mesh" / "scan7.ply"), 7, gt)
    written = io.read_mesh_ply(tmp_path / "scored" / "mesh" / "scan7.ply")[2]
    assert saved["n_faces"] == len(written) and saved["n_samples"] > 0 and saved["n_acc"] > 0
    assert _drop_time(saved) == json.loads(json.dumps(_drop_time(again)))
    assert _drop_time(outs["scored"][3]) == _drop_time(again)


def test_eval_pipeline_mesh_score_colmap_tnt_route(tmp_path, capsys):
    root = tmp_path / "Barn"
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
              "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0", "--ckpt", str(ckpt),
              "--tnt_gt", str(gt), "--tnt_tau", "0.04", "--mesh"]
    ep.main(common + ["--out", str(tmp_path / "plain")])
    capsys.readouterr()
    ep.main(common + ["--out", str(tmp_path / "scored"), "--mesh_score"])
    printed = capsys.readouterr().out
    assert sum(ln.startswith("mesh Barn:") for ln in printed.splitlines()) == 1
    plain, scored = _tree(tmp_path / "plain"), _tree(tmp_path / "scored")
    key = os.path.join("mesh", "Barn_tnt.json")
    assert os.path.join("points", "Barn_tnt.json") in plain
    assert {k: v for k, v in scored.items() if k != key} == plain
    saved = json.loads((tmp_path / "scored" / key).read_text())
    again = tnt_eval.evaluate_mesh(str(tmp_path / "scored" / "mesh" / "Barn.ply"),
                                   str(tmp_path / "scored" / "Barn"), str(gt), "Barn", tau=0.04)
    assert saved["n_samples"] > 0 and saved["spacing"] == 0.01
    assert _drop_time(saved) == json.loads(json.dumps(_drop_time(again)))


# ------------------------------------------------------------------------------ refusals
def test_budget_and_size_refusals_fire_before_the_samples_are_allocated():
    v, f = _sphere_mesh()
    V, F = _cuda(v), _cuda(f)
    n, cnt, _ = mesh_sample.sample_counts(V, F, 0.002)
    S = int(cnt.sum())
    del n, cnt
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with pytest.raises(_lib.CasMVSError, match=f"{S} surface samples needs {S * mesh_sample.BYTES_PER_SAMPLE} "
                                               "bytes.*but 1000000 bytes are available"):
        mesh_sample.sample_surface(V, F, 0.002, max_bytes=1_000_000)
    assert torch.cuda.max_memory_allocated() - base < len(f) * 64 < S * 12
    huge = _cuda(np.float32([[0, 0, 0], [1e6, 0, 0], [0, 1e6, 0]]))
    tri = _cuda(np.int32([[0, 1, 2]]))
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match="2147581953 samples"):
        mesh_sample.sample_surface(huge, tri, 1.0)
    assert torch.cuda.max_memory_allocated() - base < 1 << 20
    with pytest.raises(ValueError, match="no faces"):
        dtu_eval.evaluate_mesh((V, F[:0]), 1, os.path.dirname(__file__))
