"""Poisson surface reconstruction on the GPU (csrc/poisson.cu through poisson.py): every stage
against the float64 restatement at depth 6 on a sphere, a plane and a DTU-like scan cloud, then
end to end: deterministic bytes, a dense sphere at depth 9, the memory refusal, the command line
and eval_pipeline --mesh --mesh_method poisson."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, mesh, poisson, synth_dtu, synth_scenes
from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import io as cio
from oracle import mesh_oracle as M
from oracle import poisson_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cuda(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _cloud(kind):
    """-> (xyz, rgb, normals or None, cameras or None)"""
    rng = np.random.default_rng(5)
    if kind == "sphere":
        p, n = O.sphere(20_000, seed=0, noise=0.002)
        return p, rng.integers(0, 256, (len(p), 3)).astype(np.uint8), n, None
    if kind == "plane":
        p, n = O.plane(20_000, seed=1, noise=0.002)
        n = n.copy()
        n[:50] = 0                                             # zero-length normals are dropped
        return p, None, n, None
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        p = synth_dtu.make_scene(d, n_stl=2000, n_data=40_000, seed=2)
    cams = synth_dtu.CENTER + np.array([[0, 0, -500.0], [80, 0, -480], [-80, 40, -490]])
    return p, rng.integers(0, 256, (len(p), 3)).astype(np.uint8), None, cams


@pytest.fixture(scope="module", params=["sphere", "plane", "dtu"])
def stages(request):
    p, rgb, n, cams = _cloud(request.param)
    want = O.poisson(p, rgb, n, cams, depth=6)
    got = {}
    out = poisson.poisson_mesh(_cuda(p), _cuda(rgb), _cuda(n), cams, depth=6, fields=got)
    got = {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in got.items()}
    return want, got, out


def test_kept_points_and_normals(stages):
    want, got, (_, _, _, st) = stages
    idx = got["index"]
    assert np.array_equal(np.sort(idx), np.nonzero(want["kept"])[0])
    assert st["dropped"] == want["dropped"] and st["points"] == len(idx)
    full = np.zeros((len(want["kept"]), 3), np.float32)
    full[want["kept"]] = want["normals"]
    assert np.abs(got["normals"] - full[idx]).max() <= 1e-6


def test_splat_fields_and_divergence(stages):
    want, got, _ = stages
    N = want["grid"]["N"]
    for k, shape in (("V", (N, N, N, 3)), ("W", (N, N, N)), ("C", (N, N, N, 3)), ("b", (N, N, N))):
        g, w = got[k].reshape(shape).astype(np.float64), want[k]
        assert np.abs(g - w).max() <= 1e-5 * np.abs(w).max(), k


def test_solve_iso_level_and_trim(stages):
    want, got, (_, _, _, st) = stages
    N = want["grid"]["N"]
    chi, wchi = got["chi"].reshape(N, N, N), want["chi"]
    scale = np.abs(wchi).max()
    assert np.abs(chi - wchi).max() <= 1e-4 * scale
    assert abs(got["iso"] - want["iso"]) <= 1e-5 * scale
    assert st["residual"] <= 1e-5 and st["cycles"] <= 10
    assert abs(st["cycles"] - want["cycles"]) <= 1
    assert np.array_equal(got["keep"].reshape(N, N, N).astype(bool), want["keep"])


def test_colour_bricks_and_mesh(stages):
    want, got, (verts, colours, faces, st) = stages
    assert np.array_equal(got["keys"], want["keys"]) and st["bricks"] == len(want["keys"])
    assert np.array_equal(got["weight"], want["weight"])
    col = got["color"].reshape(-1, 3).astype(np.float64)
    assert np.abs(col - want["color"]).max() <= 1e-5 * max(1.0, np.abs(want["color"]).max())
    scale = np.abs(want["chi"]).max()
    assert np.abs(got["tsdf"].astype(np.float64) - want["tsdf"]).max() <= 1e-4 * scale
    # the same surface: sign flips of f within the solver's tolerance move a handful of cells
    # (the DTU-like cloud's outliers stretch its depth-6 grid, so its mesh is small)
    for g, w in ((len(verts), len(want["verts"])), (len(faces), len(want["faces"]))):
        assert w > 50 and abs(g - w) <= max(2, 0.005 * w)


def test_two_runs_write_the_same_bytes(tmp_path):
    views = synth_scenes.sphere_scene(8, (320, 240), seed=1, device=DEV)
    p = torch.cat([v["points"] for v in views])
    rgb = torch.cat([v["image"][v["depth"] > 0] for v in views]).to(torch.uint8)
    cams = np.stack([-np.linalg.inv(v["P"][:3, :3].astype(np.float64)) @ v["P"][:3, 3] for v in views])
    paths = []
    for i in range(2):
        v, c, f, st = poisson.poisson_mesh(p, rgb, cam_centres=cams, depth=8)
        paths.append(tmp_path / f"m{i}.ply")
        mesh.write_mesh_ply(paths[-1], v, c, f)
    assert len(f) > 10_000 and st["dropped"] < len(p) // 100
    assert paths[0].read_bytes() == paths[1].read_bytes()


def test_dense_sphere_at_depth_9_is_closed_and_within_one_node():
    p, n = O.sphere(2_000_000, seed=4)
    v, _, f, st = poisson.poisson_mesh(_cuda(p), normals=_cuda(n), depth=9)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    d = np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - 1.0)
    assert st["dropped"] == 0 and st["residual"] <= 1e-5
    assert d.max() < 1.0 * st["h"]
    assert M.is_closed_oriented(f) and M.euler_characteristic(len(v), f) == 2
    assert M.signed_volume(v, f) > 0


def test_a_grid_that_does_not_fit_is_refused_with_a_depth_that_would():
    p, n = O.sphere(10_000, seed=6)
    budget = poisson._bytes_needed(8, len(p)) - 1
    with pytest.raises(_lib.CasMVSError, match="depth 7 would fit"):
        poisson.poisson_mesh(_cuda(p), normals=_cuda(n), depth=9, max_bytes=budget)
    _, _, f, st = poisson.poisson_mesh(_cuda(p), normals=_cuda(n), depth=7, max_bytes=budget)
    assert len(f) > 0 and st["N"] == 128


def test_bricks_that_do_not_fit_are_refused_with_a_depth_that_would():
    # a volume-filling cloud: the trim keeps nearly every node, so bricks fill the grid
    rng = np.random.default_rng(8)
    p = rng.uniform(-1, 1, (20_000, 3)).astype(np.float32)
    n = rng.normal(size=(20_000, 3)).astype(np.float32)
    budget = poisson._bytes_needed(7, len(p)) + (1 << 20)
    with pytest.raises(_lib.CasMVSError, match="bricks .* depth 6 would fit"):
        poisson.poisson_mesh(_cuda(p), normals=_cuda(n), depth=7, max_bytes=budget)
    _, _, f, st = poisson.poisson_mesh(_cuda(p), normals=_cuda(n), depth=6, max_bytes=budget)
    assert st["N"] == 64 and st["bricks"] > 0


def test_command_line_with_ply_normals_and_with_cameras(tmp_path, capsys):
    from casmvsnet_pl_b200 import fusion
    views = synth_scenes.sphere_scene(6, (160, 120), seed=3, plane=False, device=DEV)
    pts = torch.cat([v["points"] for v in views]).cpu().numpy()
    fusion.write_ply(str(tmp_path / "cloud.ply"), pts, np.full((len(pts), 3), 200, np.uint8))
    cams = tmp_path / "cams"
    cams.mkdir()
    K = np.array([[0.9 * 160, 0, 80], [0, 0.9 * 160, 60], [0, 0, 1]])
    for i, v in enumerate(views):
        E = np.eye(4)
        E[:3] = np.linalg.inv(K) @ v["P"][:3].astype(np.float64)
        with open(cams / f"{i:08d}_cam.txt", "w") as f:
            f.write("extrinsic\n" + "\n".join(" ".join(f"{x:.9g}" for x in r) for r in E) +
                    "\n\nintrinsic\n" + "\n".join(" ".join(f"{x:.9g}" for x in r) for r in K) +
                    "\n\n2.0 0.01\n")
    poisson.main(["--ply", str(tmp_path / "cloud.ply"), "--out", str(tmp_path / "m.ply"),
                  "--cams", str(cams), "--depth", "7"])
    assert "triangles" in capsys.readouterr().out
    v, c, f = cio.read_mesh_ply(str(tmp_path / "m.ply"))
    assert len(f) > 1000 and (c == 200).all()
    assert M.signed_volume(v, f) > 0                          # oriented outward by the cameras
    p, n = O.sphere(20_000, seed=7)
    v = np.empty(len(p), dtype=[(k, "<f4") for k in ("x", "y", "z", "nx", "ny", "nz")])
    for a, k in enumerate("xyz"):
        v[k], v["n" + k] = p[:, a], n[:, a]
    with open(tmp_path / "n.ply", "wb") as fh:
        fh.write((f"ply\nformat binary_little_endian 1.0\nelement vertex {len(p)}\n" +
                  "".join(f"property float {k}\n" for k in v.dtype.names) + "end_header\n").encode())
        v.tofile(fh)
    poisson.main(["--ply", str(tmp_path / "n.ply"), "--out", str(tmp_path / "n_mesh.ply"),
                  "--depth", "6"])
    v, c, f = cio.read_mesh_ply(str(tmp_path / "n_mesh.ply"))
    assert M.is_closed_oriented(f) and (c == 255).all()


def _tree_bytes(d):
    return {os.path.relpath(os.path.join(r, n), d): open(os.path.join(r, n), "rb").read()
            for r, _, files in os.walk(d) for n in files}


def test_eval_pipeline_poisson_mesh_end_to_end(tmp_path, capsys):
    from casmvsnet_pl_b200 import ABN, synth
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    root = tmp_path / "capture"
    synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), n_points=3000, seed=7)
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN)
    synth.randomize_model_(model, 0)
    ckpt = tmp_path / "weights.pt"
    torch.save(model.state_dict(), ckpt)
    common = ["--dataset_name", "colmap", "--root_dir", str(root), "--img_wh", "128", "96",
              "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0", "--ckpt", str(ckpt)]
    poisson_flags = ["--mesh", "--mesh_method", "poisson", "--poisson_depth", "7"]
    for tag, extra in (("plain", []), ("p1", poisson_flags), ("p2", poisson_flags)):
        ep.main(common + ["--out", str(tmp_path / tag)] + extra)
    assert "capture: poisson mesh at depth 7" in capsys.readouterr().out
    plain, m1, m2 = (_tree_bytes(tmp_path / t) for t in ("plain", "p1", "p2"))
    mesh_file = os.path.join("mesh", "capture.ply")
    assert m1[mesh_file] == m2[mesh_file]
    assert {k: v for k, v in m1.items() if k != mesh_file} == plain
    v, _, f = cio.read_mesh_ply(str(tmp_path / "p1" / mesh_file))
    assert len(f) > 0 and f.min() >= 0 and f.max() < len(v)
