"""Rendering on the GPU (csrc/render.cu through render.py): images and depth maps bit-identical to
the numpy restatement for clouds, scene meshes and random triangles, reproducible across buffers,
rendered depth against the analytic depth of a synthetic scene, and the command line end to end
after eval_pipeline --mesh."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, mesh, render, synth_scenes
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import render_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def no_fallbacks():
    n0 = _lib.fallback_count()
    yield
    assert _lib.fallback_count() == n0


def _same(got, want):
    img, depth = (t.cpu().numpy() for t in got)
    assert np.array_equal(img, want[0])
    assert np.array_equal(depth.view(np.uint32), want[1].view(np.uint32))


def _look_at_P(C, target, wh, f_scale=0.9):
    W, H = wh
    R = synth_scenes._look_at(np.asarray(C, float), np.asarray(target, float))
    K = np.array([[f_scale * W, 0, W / 2 - 0.5], [0, f_scale * W, H / 2 - 0.5], [0, 0, 1]])
    E = np.eye(4)
    E[:3, :3], E[:3, 3] = R, -R @ np.asarray(C, float)
    return render.projection(K, E).astype(np.float32)


def _random_cloud(n, wh, seed):
    """n points around the origin seen by a camera 4 units away, with exact duplicates (depth
    ties), points behind the camera, NaN / inf coordinates and points far off-screen."""
    rng = np.random.default_rng(seed)
    xyz = rng.normal(0, 1, (n, 3)).astype(np.float32)
    dup = rng.choice(n, n // 10, replace=False)
    xyz[dup] = xyz[rng.choice(n, n // 10)]                   # ties at the same pixel and depth
    k = rng.choice(n, n // 50, replace=False)
    xyz[k[: len(k) // 3]] = [0.0, 0.0, 9.0]                  # behind the camera (at z = 4)
    xyz[k[len(k) // 3: 2 * len(k) // 3], rng.integers(0, 3)] = np.nan
    xyz[k[2 * len(k) // 3:], 0] = rng.choice([np.inf, 40.0, -40.0], len(k) - 2 * len(k) // 3)
    rgb = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    P = _look_at_P([0.3, -0.2, 4.0], [0.0, 0.1, 0.0], wh)
    return xyz, rgb, P


@pytest.mark.parametrize("size", [1, 3])
def test_points_equal_the_restatement(size):
    wh = (640, 480)
    xyz, rgb, P = _random_cloud(1_000_000, wh, seed=size)
    got = render.render_points(torch.from_numpy(xyz).to(DEV), torch.from_numpy(rgb).to(DEV), P, wh, size)
    want = O.render_points(xyz, rgb, P, wh, size)
    _same(got, want)
    assert (want[1] > 0).sum() > 0.3 * wh[0] * wh[1]
    # the duplicates do tie: some pixel is won by the lower of two identical points
    idx = (want[2][want[2] != O.EMPTY] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    _, first = np.unique(xyz, axis=0, return_index=True)
    assert np.isin(idx, first).all()


def test_two_calls_on_differently_offset_buffers_are_equal():
    wh = (333, 250)
    xyz, rgb, P = _random_cloud(200_000, wh, seed=5)
    a = render.render_points(torch.from_numpy(xyz).to(DEV), torch.from_numpy(rgb).to(DEV), P, wh, 2)
    big = torch.zeros(len(xyz) * 3 + 5, device=DEV)
    x2 = big[5:].view(-1, 3)
    x2.copy_(torch.from_numpy(xyz))
    cbig = torch.zeros(len(rgb) * 3 + 7, dtype=torch.uint8, device=DEV)
    c2 = cbig[7:].view(-1, 3)
    c2.copy_(torch.from_numpy(rgb))
    torch.cuda.empty_cache()
    b = render.render_points(x2, c2, P, wh, 2)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.fixture(scope="module")
def scene_mesh():
    views = synth_scenes.sphere_scene(8, (320, 240), seed=11, device=DEV)
    verts, cols, faces, st = mesh.mesh_views([v["points"] for v in views],
                                             [v["depth"] for v in views],
                                             [v["image"] for v in views], [v["P"] for v in views])
    return views, verts, cols, faces, st


@pytest.mark.parametrize("view", ["default", "close_up"])
def test_scene_mesh_equals_the_restatement(scene_mesh, view):
    _, verts, cols, faces, _ = scene_mesh
    wh = (640, 480)
    if view == "default":
        P = render.projection(*render.default_view(verts, wh)).astype(np.float32)
    else:
        P = _look_at_P(1.5 * np.array([0.6, 0.5, 0.62]), [0.0, 0.0, 0.0], wh)
    v, c, f = (t.cpu().numpy() for t in (verts, cols, faces))
    drawn, bw, bh = O.projected_boxes(v, f, P, wh)
    big = drawn & ((bw > O.SMALL_BOX) | (bh > O.SMALL_BOX))
    if view == "close_up":
        assert big.sum() > 1000                                  # the CTA path is exercised
    else:
        assert (drawn & ~big).sum() > 1000
    got = render.render_mesh(verts, cols, faces, P, wh)
    want = O.render_mesh(v, c, f, P, render.camera_centre(P), wh)
    _same(got, want)
    assert (want[1] > 0).sum() > 0.1 * wh[0] * wh[1]
    again = render.render_mesh(verts.clone(), cols.clone(), faces.clone(), P, wh)
    assert torch.equal(again[0], got[0]) and torch.equal(again[1], got[1])


def test_random_large_and_degenerate_triangles_equal_the_restatement():
    rng = np.random.default_rng(3)
    wh = (320, 240)
    P = _look_at_P([0.0, 0.0, 5.0], [0.0, 0.0, 0.0], wh)
    n = 3000
    v = rng.normal(0, 1.0, (n, 3)).astype(np.float32)
    v[:30] *= 4                                                    # screen-filling triangles
    v[30:60, 2] = 5.5                                              # behind the camera
    v[60:70] = np.nan
    v[300:400] = 2 * v[200:300] - v[100:200]                       # collinear with 100.., 200..
    c = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    f = rng.integers(0, n, (3000, 3)).astype(np.int32)
    f[:200, 1] = f[:200, 0]                                        # repeated vertex: zero area
    f[200:300] = np.arange(100, 400).reshape(3, 100).T
    f[300:330] = rng.integers(0, 30, (30, 3))
    got = render.render_mesh(*(torch.from_numpy(a).to(DEV) for a in (v, c, f)), P, wh)
    want = O.render_mesh(v, c, f, P, render.camera_centre(P), wh)
    _same(got, want)
    drawn, bw, bh = O.projected_boxes(v, f, P, wh)
    assert (drawn & (bw * bh > 20_000)).sum() > 10


def test_bad_face_index_is_refused():
    v = torch.zeros(4, 3, device=DEV)
    v[:, 2] = 1
    c = torch.zeros(4, 3, dtype=torch.uint8, device=DEV)
    P = np.eye(4, dtype=np.float32)
    for bad in (4, -1):
        f = torch.tensor([[0, 1, 2], [0, bad, 3]], dtype=torch.int32, device=DEV)
        with pytest.raises(_lib.CasMVSError, match="face index"):
            render.render_mesh(v, c, f, P, (16, 16))
    img, depth = render.render_mesh(v, c, torch.tensor([[0, 1, 2]], dtype=torch.int32, device=DEV), P,
                                    (16, 16))
    assert (img.cpu().numpy() == O.BACKGROUND).all() and (depth == 0).all()   # zero area


def test_rendered_depth_matches_the_analytic_depth(scene_mesh):
    views, verts, cols, faces, st = scene_mesh
    v = views[0]
    H, W = v["depth"].shape
    D = v["depth"].cpu().numpy()
    rgb = v["image"][v["depth"] > 0].round().to(torch.uint8)
    _, depth = render.render_points(v["points"], rgb, v["P"], (W, H))
    R = depth.cpu().numpy()
    hit = D > 0
    exact = hit & (np.abs(R - D) <= D * 2.0 ** -20)
    frac = exact.sum() / hit.sum()
    worst = np.abs(R - D)[hit].max()
    print(f"own points: {frac:.5f} of {hit.sum()} surface pixels at the analytic depth, "
          f"worst {worst:.3g}; drawn off the surface: {(R[~hit] > 0).sum()}")
    assert frac >= 0.99
    # the TSDF mesh: interior surface pixels (5x5 neighbourhood on the surface, no depth jump)
    _, mdepth = render.render_mesh(verts, cols, faces, v["P"], (W, H))
    M = mdepth.cpu().numpy()
    pad = np.pad(D, 2)
    win = np.stack([pad[dy:dy + H, dx:dx + W] for dy in range(5) for dx in range(5)])
    interior = (win > 0).all(0) & (win.max(0) - win.min(0) < 4 * st["voxel"])
    err = np.abs(M - D)[interior]
    within = (err <= st["voxel"]).mean()
    print(f"mesh: {within:.5f} of {interior.sum()} interior pixels within one voxel "
          f"({st['voxel']:.4g}); worst {err.max():.3g}")
    assert interior.sum() > 0.2 * hit.sum() and within >= 0.99


def _tree_bytes(d):
    return {os.path.relpath(os.path.join(r, n), d): open(os.path.join(r, n), "rb").read()
            for r, _, files in os.walk(d) for n in files}


def test_cli_end_to_end_after_eval_pipeline_mesh(tmp_path, capsys):
    from PIL import Image

    from casmvsnet_pl_b200 import ABN, synth
    from casmvsnet_pl_b200 import io as cio
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    root = tmp_path / "capture"
    synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), n_points=3000, seed=7)
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN)
    synth.randomize_model_(model, 0)
    ckpt = tmp_path / "weights.pt"
    torch.save(model.state_dict(), ckpt)
    common = ["--dataset_name", "colmap", "--root_dir", str(root), "--img_wh", "128", "96",
              "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0", "--ckpt", str(ckpt),
              "--mesh"]
    for tag in ("a", "b"):
        ep.main(common + ["--out", str(tmp_path / tag)])
    plain = _tree_bytes(tmp_path / "b")
    out = tmp_path / "a"
    base = ["--dataset_name", "colmap", "--scan", "capture", "--out", str(out)]
    pngs = {}
    for name, extra in (("save", ["--save_viewpoint"]), ("use", ["--use_viewpoint"]),
                        ("mesh", ["--use_viewpoint", "--mesh"])):
        png = render.main(base + extra)
        pngs[name] = np.asarray(Image.open(png))
    log = capsys.readouterr().out
    assert "capture contains" in log and "pixels drawn" in log and "triangles" in log
    xyz, rgb, _ = render.load_scan(str(out / "points" / "capture.ply"), False)
    P, wh = render.read_viewpoint(str(out / "viewpoint.json"))
    assert wh == render.DEFAULT_WH
    want = O.render_points(xyz, rgb, P, wh)[0]
    assert np.array_equal(pngs["save"], want) and np.array_equal(pngs["use"], want)
    mv, mc, mf = cio.read_mesh_ply(str(out / "mesh" / "capture.ply"))
    want_m = O.render_mesh(mv, mc, mf, P, render.camera_centre(P), wh)[0]
    assert np.array_equal(pngs["mesh"], want_m) and (want_m != O.BACKGROUND).any()
    again = np.asarray(Image.open(render.main(base + ["--use_viewpoint", "--mesh"])))
    assert np.array_equal(again, pngs["mesh"])                       # identical pixels
    after = _tree_bytes(out)
    extra = {k for k in after if k.startswith("render" + os.sep) or k == "viewpoint.json"}
    assert {k: v for k, v in after.items() if k not in extra} == plain   # eval outputs untouched
