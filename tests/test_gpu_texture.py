"""Mesh texturing on the GPU (texture.py, csrc/texture.cu, render.render_textured_mesh): every
stage bit for bit against the numpy restatement (oracle/texture_oracle.py) on three meshes, the
textured resolve, occlusion, byte reproducibility, fidelity against flat vertex colours, the
refusals, the command line and eval_pipeline --mesh_texture end to end."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, io, mesh, render, simplify, synth_scenes, texture
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import simplify_oracle as S
from oracle import texture_oracle as T

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _host(t):
    return t.cpu().numpy()


_SCENES = {}


def _scene(n_views=12, wh=(240, 180), voxel=0.05):
    """sphere_scene views (photos rounded to uint8 once) and their TSDF mesh (host arrays)."""
    key = (n_views, wh, voxel)
    if key not in _SCENES:
        views = synth_scenes.sphere_scene(n_views, wh, seed=3, device=DEV)
        v, c, f, _ = mesh.mesh_views([x["points"] for x in views], [x["depth"] for x in views],
                                     [x["image"] for x in views], [x["P"] for x in views], voxel=voxel)
        photos = [x["image"].round().clamp(0, 255).to(torch.uint8).cpu().numpy() for x in views]
        _SCENES[key] = (views, photos, (_host(v), _host(c), _host(f)))
    return _SCENES[key]


def _decimated(ratio):
    _, _, (v, c, f) = _scene()
    V, C, F, _ = simplify.simplify_mesh(_cuda(v), _cuda(c), _cuda(f), max(1, round(ratio * len(f))))
    return _host(V), _host(C), _host(F)


def _degenerate():
    v, f = S.grid_mesh(12)                                   # the unit square of z = 0
    n = len(v)
    extra_v = np.array([[0.5, 0.5, 0.3], [1.3, 1.3, 0.0], [1.3, 1.1, 0.0], [1.1, 1.3, 0.1]],
                       np.float32)
    a, b = 3 * 13 + 3, 3 * 13 + 4
    corner = 12 * 13 + 12
    extra_f = np.array([[a, b, n], [corner, n + 1, n + 2], [n + 1, n + 3, n + 2], [5, 5, 6],
                        [0, 1, 2]], np.int32)
    v = np.concatenate([v, extra_v]) - np.float32([0.5, 0.5, 0.0])
    c = (np.arange(3 * (n + 4)) % 251).astype(np.uint8).reshape(-1, 3)
    return v, c, np.concatenate([f, extra_f])


MESHES = {"tsdf": lambda: _scene()[2], "decimated_2pct": lambda: _decimated(0.02),
          "degenerate": _degenerate}


def _run(v, c, f, photos, Ps, **kw):
    return texture.texture_mesh(_cuda(v), _cuda(c), _cuda(f), [_cuda(p) for p in photos], Ps, **kw)


@pytest.mark.parametrize("name", list(MESHES))
def test_every_stage_is_bit_identical_to_the_oracle(name):
    views, photos, _ = _scene()
    v, c, f = MESHES[name]()
    Ps = [x["P"] for x in views]
    o = T.texture_mesh(v, c, f, photos, Ps)
    vg, fg = _cuda(v), _cuda(f).int()
    ims = [_cuda(p) for p in photos]
    score, view = texture.candidates(vg, fg, ims, Ps)
    assert np.array_equal(_host(view), o["view"])
    assert np.array_equal(_host(score).view(np.uint32), o["score"].view(np.uint32))
    nbr = texture.neighbours(fg)
    assert np.array_equal(_host(nbr), o["nbr"])
    lab0 = view[:, 0].contiguous()
    lab = texture.smooth(nbr, score, view, lab0)
    assert np.array_equal(_host(lab), o["labels"])
    comp0, _ = texture.components(nbr, lab0)
    comp, _ = texture.components(nbr, lab)
    assert np.array_equal(_host(comp0), o["comp0"]) and np.array_equal(_host(comp), o["comp"])
    uv, page, atlas, st = _run(v, c, f, photos, Ps)
    assert np.array_equal(_host(atlas), o["atlas"])
    assert np.array_equal(_host(page), o["page"])
    assert np.array_equal(_host(uv).view(np.uint32), o["uv"].view(np.uint32))
    roots = o["charts"][:, 0]
    view_charts = o["charts"][:, 1] >= 0
    assert np.array_equal(o["charts"][view_charts, 2:6], o["rect"][roots[view_charts]])
    assert st["charts"] == len(o["charts"]) and st["charts_unsmoothed"] == int(
        (o["comp0"] == np.arange(len(f))).sum())
    assert st["pages"] == len(o["atlas"]) and st["page_side"] == o["S"]
    print(f"{name}: {st}")
    if name == "tsdf":
        assert st["unseen_faces"] < 0.2 * len(f) and st["charts"] < st["charts_unsmoothed"]
    P = views[0]["P"]
    img, dep = render.render_textured_mesh(vg, fg, uv, page, atlas, P, (240, 180))
    oimg, odep = T.render_textured_mesh(v, f, o["uv"], o["page"], o["atlas"], P, (240, 180))
    assert np.array_equal(_host(img), oimg)
    assert np.array_equal(_host(dep).view(np.uint32), odep.view(np.uint32))


def _hidden_plane_faces(v, f, eye, radius=1.0, margin=0.9):
    """Faces on the plane z = -radius whose three vertices the sphere hides from `eye`, with the
    sight line passing within margin x radius of the centre."""
    x = v[f].astype(np.float64)                               # (F,3,3)
    on_plane = np.abs(x[:, :, 2] + radius).max(1) < 1e-3
    d = x - eye
    t = np.clip(-(eye[None, None] * d).sum(-1) / (d * d).sum(-1), 0, 1)
    closest = eye + t[..., None] * d
    inside = (np.linalg.norm(closest, axis=-1) < margin * radius) & (t > 0.05) & (t < 0.95)
    return np.nonzero(on_plane & inside.all(1))[0]


def test_no_hidden_plane_face_takes_a_view_that_cannot_see_it():
    views, photos, (v, c, f) = _scene()
    Ps = [x["P"] for x in views]
    score, view = texture.candidates(_cuda(v), _cuda(f).int(), [_cuda(p) for p in photos], Ps)
    view = _host(view)
    checked = 0
    for i, P in enumerate(Ps):
        hid = _hidden_plane_faces(v, f, texture.eye_of(P))
        checked += len(hid)
        assert not (view[hid] == i).any(), i
    assert checked > 100, checked


def test_two_runs_write_the_same_bytes_and_the_cli_agrees(tmp_path):
    views, photos, (v, c, f) = _scene()
    Ps = [x["P"] for x in views]
    out = []
    for i in range(2):
        uv, page, atlas, _ = _run(v, c, f, photos, Ps)
        (tmp_path / f"run{i}").mkdir()
        paths = texture.write_textured_obj(tmp_path / f"run{i}" / "m.obj", v, f, uv, page, atlas)
        out.append([open(p, "rb").read() for p in paths])
    assert out[0] == out[1]
    # the command line: cameras as MVSNet cam files, images as PNGs paired by view_names.txt
    (tmp_path / "cams").mkdir()
    (tmp_path / "imgs").mkdir()
    from PIL import Image
    W, H = 240, 180
    K = np.array([[0.9 * W, 0, W / 2], [0, 0.9 * W, H / 2], [0, 0, 1]])
    names = []
    for i, (x, p) in enumerate(zip(views, photos)):
        E = np.eye(4)
        E[:3] = np.linalg.inv(K) @ x["P"].astype(np.float64)[:3]
        with open(tmp_path / "cams" / f"{i:08d}_cam.txt", "w") as fh:
            fh.write("extrinsic\n" + "\n".join(" ".join(repr(float(a)) for a in r) for r in E)
                     + "\n\nintrinsic\n" + "\n".join(" ".join(repr(float(a)) for a in r) for r in K)
                     + "\n\n1 1\n")
        names.append(f"view_{100 - i:03d}.png")
        Image.fromarray(p).save(tmp_path / "imgs" / names[-1])
    with open(tmp_path / "view_names.txt", "w") as fh:
        fh.write("".join(f"{i} {n}\n" for i, n in enumerate(names)))
    mesh.write_mesh_ply(tmp_path / "in.ply", v, c, f)
    texture.main(["--ply", str(tmp_path / "in.ply"), "--cams", str(tmp_path / "cams"), "--images",
                  str(tmp_path / "imgs"), "--view_names", str(tmp_path / "view_names.txt"),
                  "--out", str(tmp_path / "cli.obj")])
    paths, Pc = texture.read_views(str(tmp_path / "cams"), str(tmp_path / "imgs"),
                                   str(tmp_path / "view_names.txt"))
    uv, page, atlas, st = _run(v, c, f, photos, Pc)
    texture.write_textured_obj(tmp_path / "api.obj", v, f, uv, page, atlas)
    assert (tmp_path / "cli.obj").read_bytes() == (tmp_path / "api.obj").read_bytes().replace(
        b"api", b"cli")
    assert (tmp_path / "cli_0.png").read_bytes() == (tmp_path / "api_0.png").read_bytes()
    assert st["unseen_faces"] < 0.2 * len(f)


def test_textured_rendering_is_far_closer_to_the_photos_than_vertex_colours():
    views, photos, (v, c, f) = _scene(12, (480, 360), 0.02)
    V, C, F = _host_decimate(v, c, f, 0.01)
    Ps = [x["P"] for x in views]
    tex = _run(V, C, F, photos, Ps)
    flat = _run(V, C, F, [], [])
    assert flat[3]["flat_charts"] == len(F) and flat[3]["views"] == 0
    err = {}
    for name, (uv, page, atlas, st) in (("textured", tex), ("flat", flat)):
        tot = n = 0
        for x, p in zip(views[:6], photos[:6]):
            img, dep = render.render_textured_mesh(_cuda(V), _cuda(F).int(), uv, page, atlas, x["P"],
                                                   (480, 360))
            both = (_host(dep) > 0) & (x["depth"].cpu().numpy() > 0)
            tot += np.abs(_host(img).astype(np.int64) - p.astype(np.int64))[both].sum()
            n += 3 * both.sum()
        err[name] = tot / n
    print(f"mean absolute error over {len(F)} faces: textured {err['textured']:.3f}, "
          f"flat {err['flat']:.3f}; stats {tex[3]}")
    # measured on an H100: textured 4.965, flat 35.730
    assert err["textured"] < 0.25 * err["flat"]


def _host_decimate(v, c, f, ratio):
    V, C, F, _ = simplify.simplify_mesh(_cuda(v), _cuda(c), _cuda(f), max(1, round(ratio * len(f))))
    return _host(V), _host(C), _host(F)


def test_bad_inputs_and_oversized_work_are_refused():
    views, photos, _ = _scene()
    v, c, f = _degenerate()
    Ps = [views[0]["P"]]
    ims = [photos[0]]
    bad_v = v.copy()
    bad_v[3, 1] = np.inf
    with pytest.raises(ValueError, match="non-finite"):
        _run(bad_v, c, f, ims, Ps)
    bad_f = f.copy()
    bad_f[2, 0] = len(v)
    with pytest.raises(ValueError, match="outside"):
        _run(v, c, bad_f, ims, Ps)
    with pytest.raises(ValueError, match="uint8 CUDA tensor"):
        texture.texture_mesh(_cuda(v), _cuda(c), _cuda(f), [_cuda(photos[0]).float()], Ps)
    with pytest.raises(ValueError, match="uint8 CUDA tensor"):
        texture.texture_mesh(_cuda(v), _cuda(c), _cuda(f), [_cuda(photos[0][..., :2])], Ps)
    with pytest.raises(ValueError, match="finite 4x4"):
        _run(v, c, f, ims, [np.full((4, 4), np.nan, np.float32)])
    with pytest.raises(ValueError, match="finite 4x4"):
        _run(v, c, f, ims, [np.eye(3, dtype=np.float32)])
    with pytest.raises(ValueError, match="1 images but 2"):
        _run(v, c, f, ims, Ps * 2)
    with pytest.raises(_lib.CasMVSError, match="needs .* bytes .* but 1000 bytes"):
        _run(v, c, f, ims, Ps, max_bytes=1000)


def _tree_bytes(d):
    return {os.path.relpath(os.path.join(r, n), d): open(os.path.join(r, n), "rb").read()
            for r, _, files in os.walk(d) for n in files}


def test_eval_pipeline_mesh_texture_end_to_end(tmp_path):
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
              "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0", "--ckpt", str(ckpt),
              "--mesh", "--mesh_faces", "300"]
    ep.main(common + ["--out", str(tmp_path / "plain")])
    ep.main(common + ["--mesh_texture", "--out", str(tmp_path / "tex")])
    plain, tex = _tree_bytes(tmp_path / "plain"), _tree_bytes(tmp_path / "tex")
    ply = os.path.join("mesh", "capture.ply")
    assert tex[ply] == plain[ply]
    extra = sorted(set(tex) - set(plain))
    assert extra[:2] == [os.path.join("mesh", "capture.mtl"), os.path.join("mesh", "capture.obj")]
    assert all(k.startswith(os.path.join("mesh", "capture_")) and k.endswith(".png") for k in extra[2:])
    assert {k: b for k, b in tex.items() if k not in extra} == plain
    V, F, uv, page, atlas = texture.read_textured_obj(tmp_path / "tex" / "mesh" / "capture.obj")
    v0, _, f0 = io.read_mesh_ply(tmp_path / "plain" / ply)
    assert np.array_equal(V, v0) and np.array_equal(F, f0) and len(F) <= 300
    assert len(atlas) == len(extra) - 2 and uv.shape == (len(F), 3, 2)
    png = render.main(["--dataset_name", "colmap", "--scan", "capture", "--mesh", "--textured",
                       "--out", str(tmp_path / "tex")])
    assert png.endswith("capture_textured.png") and os.path.isfile(png)
