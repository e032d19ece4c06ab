"""Meshing on the GPU (csrc/mesh.cu through mesh.py): brick allocation, TSDF integration and
marching-cubes extraction bit-identical to the numpy restatement, a closed sphere from views all
around, and eval_pipeline --mesh end to end on synthetic captures (deterministic, and leaving
every other output byte-identical)."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, mesh, synth_scenes
from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import io as cio
from oracle import mesh_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _scene(n_views, wh, seed, plane=True):
    return synth_scenes.sphere_scene(n_views, wh, seed=seed, plane=plane, device=DEV)


def _host_views(views):
    return [(v["depth"].cpu().numpy(), v["image"].cpu().numpy(), v["P"]) for v in views]


def test_brick_keys_match_the_restatement_and_drop_bad_points():
    views = _scene(4, (160, 120), seed=0)
    pts = torch.cat([v["points"] for v in views])
    bad = torch.tensor([[float("nan"), 0, 0], [1e9, 0, 0], [0, -1e9, 0]], device=DEV)
    pts = torch.cat([pts[:1000], bad, pts[1000:]])
    vol = mesh.TSDFVolume(pts, 0.05)
    want, dropped = O.brick_keys(pts.cpu().numpy(), vol.voxel, vol.trunc)
    assert np.array_equal(vol.keys.cpu().numpy(), want)
    assert vol.dropped == dropped == 3
    assert np.array_equal(vol.nbr.cpu().numpy(), O.brick_neighbors(want))


def test_integration_and_extraction_are_bit_identical_to_the_restatement():
    views = _scene(11, (160, 120), seed=1)                # two launches of 8 views and 3 views
    voxel = mesh.default_voxel_size([v["depth"] for v in views], [v["P"] for v in views])
    vol = mesh.TSDFVolume([v["points"] for v in views], voxel)
    vol.integrate([v["depth"] for v in views], [v["image"] for v in views], [v["P"] for v in views])
    keys = vol.keys.cpu().numpy()
    s, w, c = O.integrate(keys, _host_views(views), vol.voxel, vol.trunc)
    got = [t.cpu().numpy() for t in (vol.tsdf, vol.weight, vol.color)]
    assert (w > 0).sum() > 10_000
    for g, want in zip(got, (s, w, c)):
        assert np.array_equal(g.view(np.uint32), want.view(np.uint32))
    verts, cols, faces = vol.extract()
    ov, oc, of = O.extract(keys, s, w, c, vol.voxel)
    assert len(of) > 1000
    assert np.array_equal(verts.cpu().numpy().view(np.uint32), ov.view(np.uint32))
    assert np.array_equal(cols.cpu().numpy(), oc)
    assert np.array_equal(faces.cpu().numpy(), of)
    again = vol.extract()
    assert all(torch.equal(a, b) for a, b in zip(again, (verts, cols, faces)))


def test_view_at_a_time_equals_batched_integration():
    views = _scene(9, (128, 96), seed=2)
    pts = [v["points"] for v in views]
    a, b = mesh.TSDFVolume(pts, 0.06), mesh.TSDFVolume(pts, 0.06)
    a.integrate([v["depth"] for v in views], [v["image"] for v in views], [v["P"] for v in views])
    for v in views:
        b.integrate(v["depth"], v["image"], v["P"])
    for x, y in ((a.tsdf, b.tsdf), (a.weight, b.weight), (a.color, b.color)):
        assert torch.equal(x, y)


def test_sphere_seen_from_all_around_is_a_closed_sphere():
    views = _scene(20, (320, 240), seed=3, plane=False)
    verts, cols, faces, st = mesh.mesh_views([v["points"] for v in views],
                                             [v["depth"] for v in views],
                                             [v["image"] for v in views], [v["P"] for v in views])
    v, f = verts.cpu().numpy(), faces.cpu().numpy()
    assert st["triangles"] == len(f) > 10_000 and st["dropped"] == 0
    assert O.is_closed_oriented(f)
    assert O.euler_characteristic(len(v), f) == 2
    assert np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - 1.0).max() < st["voxel"]
    assert O.signed_volume(v, f) > 0                         # normals point out


def test_a_volume_that_does_not_fit_is_refused_with_a_voxel_size_that_would():
    views = _scene(3, (128, 96), seed=4)
    pts = [v["points"] for v in views]
    need = mesh.TSDFVolume(pts, 0.02).n_voxels * mesh.BYTES_PER_VOXEL
    with pytest.raises(_lib.CasMVSError, match="a voxel size of about") as e:
        mesh.TSDFVolume(pts, 0.02, max_bytes=need // 10)
    fit = float(str(e.value).rsplit("about ", 1)[1].split()[0])
    assert mesh.TSDFVolume(pts, fit).n_voxels * mesh.BYTES_PER_VOXEL <= need // 10


def _model():
    from casmvsnet_pl_b200 import ABN, synth
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN)
    synth.randomize_model_(model, 0)
    return model.eval().cuda()


def _tree_bytes(d):
    return {os.path.relpath(os.path.join(r, n), d): open(os.path.join(r, n), "rb").read()
            for r, _, files in os.walk(d) for n in files}


@pytest.mark.parametrize("kind", ["colmap", "tanks"])
def test_eval_pipeline_mesh_end_to_end(tmp_path, kind, capsys):
    if kind == "colmap":
        root = tmp_path / "capture"
        synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), n_points=3000, seed=7)
        args = ["--dataset_name", "colmap", "--root_dir", str(root)]
        scan = "capture"
    else:
        synth_scenes.make_tanks(str(tmp_path / "tnt"), "intermediate", "Horse", n_views=6,
                                image_wh=(200, 120), seed=3)
        args = ["--dataset_name", "tanks", "--split", "intermediate", "--scan", "Horse",
                "--root_dir", str(tmp_path / "tnt")]
        scan = "Horse"
    ckpt = tmp_path / "weights.pt"                           # the same weights for every run
    torch.save(_model().state_dict(), ckpt)
    common = args + ["--img_wh", "128", "96", "--n_views", "3", "--conf", "0",
                     "--min_geo_consistent", "0", "--ckpt", str(ckpt)]
    for tag, extra in (("plain", []), ("mesh1", ["--mesh"]), ("mesh2", ["--mesh"])):
        ep.main(common + ["--out", str(tmp_path / tag)] + extra)
    log = capsys.readouterr().out
    assert f"{scan}: mesh at voxel" in log and "triangles" in log
    plain, m1, m2 = (_tree_bytes(tmp_path / t) for t in ("plain", "mesh1", "mesh2"))
    mesh_file = os.path.join("mesh", f"{scan}.ply")
    assert m1[mesh_file] == m2[mesh_file]                    # byte-identical meshes
    assert {k: v for k, v in m1.items() if k != mesh_file} == plain   # nothing else changes
    verts, cols, faces = cio.read_mesh_ply(str(tmp_path / "mesh1" / mesh_file))
    assert len(faces) > 0 and faces.min() >= 0 and faces.max() < len(verts)
    _, uc, _, _ = O.edge_counts(faces)
    assert uc.max() <= 2                                      # no edge has more than two faces
