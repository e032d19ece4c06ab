"""Mesh refinement on the GPU (csrc/refine.cu, casmvsnet_pl_b200/refine.py) against the float64
oracle (oracle/refine_oracle.py): each kernel on the GPU's own inputs, then whole calls; two runs
give the same bits, faces and colours do not change, a textureless scene moves nothing, bad input
is refused, and eval_pipeline --mesh_refine changes only the mesh's vertices."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, io, refine, synth_scenes
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import refine_oracle as O
from oracle import texture_oracle as TO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _bumpy(n=18, z=0.03, seed=0):
    """A grid over the textured plane, lifted by z and seeded bumps of up to 2 footprints, with
    one vertex no face uses."""
    v, f = O.grid_mesh(n=n)
    rng = np.random.default_rng(seed)
    v[:, 2] = z + 0.02 * np.sin(7 * v[:, 0]) * np.cos(5 * v[:, 1]) + rng.uniform(-0.01, 0.01, len(v))
    v = np.concatenate([v, np.float32([[0.0, 0.0, 0.1]])]).astype(np.float32)
    c = (np.arange(3 * len(v)) % 251).astype(np.uint8).reshape(-1, 3)
    return v, c, f


SCENES = {"5_views": dict(), "6_views_wide": dict(spread=1.2, extra=True)}


def _views(name):
    kw = dict(SCENES[name])
    extra = kw.pop("extra", False)
    ims, Ps, srcs = O.plane_scene(**kw)
    if extra:                                 # a sixth view that no list names as a source
        ims.append(ims[0][::-1].copy())
        Ps.append(Ps[0])
        srcs = [s[::-1] for s in srcs] + [[0, 1, 2, 3, 4]]
    return ims, Ps, srcs


@pytest.mark.parametrize("name", sorted(SCENES))
def test_every_kernel_agrees_with_the_oracle(name):
    ims, Ps, srcs = _views(name)
    v, c, f = _bumpy()
    V = len(v)
    images = [_cuda(im) for im in ims]
    greys = refine.grey_images(images)
    for g, im in zip(greys, ims):
        assert np.array_equal(g.cpu().numpy(), O.grey(im))
    views = refine._device_views(images, Ps, greys)
    eyes = np.stack([TO.eye_of(P) for P in Ps])
    faces = _cuda(f)
    vf, nb = refine.topology(faces, V)
    cur = _cuda(v)
    host = v
    src_csr = refine.source_csr(srcs, len(ims), DEV)
    whs = [(im.shape[1], im.shape[0]) for im in ims]
    checked_k = 0
    for it in range(3):
        normal = refine.normals(cur, faces, vf)
        n_host = normal.cpu().numpy()
        on = O.normals(host, f)
        assert np.abs(n_host - on).max() <= 4 * O.EPS
        vis = refine.visibility(cur, faces, normal, images, Ps, eyes)
        bits = vis.cpu().numpy().view(np.uint32)
        gv = (bits[:, np.arange(len(ims)) // 32] >> (np.arange(len(ims)) % 32)) & 1
        ov = O.visibility(host, n_host, Ps, whs, [TO.key_buffer(host, f, P, wh) for P, wh in
                                                  zip(Ps, whs)], eyes)
        assert np.array_equal(gv.astype(bool), ov)
        ref, src = refine.select(cur, normal, vis, _cuda(eyes), src_csr)
        oref, osrc = O.select(host, n_host, ov, eyes, srcs)
        assert np.array_equal(ref.cpu().numpy(), oref) and np.array_equal(src.cpu().numpy(), osrc)
        assert (oref >= 0).sum() > 0.7 * V
        sw = refine.sweep(cur, normal, ref, src, views, it, want_scores=True)
        g = {k: t.cpu().numpy() for k, t in sw.items()}
        o = O.sweep(host, n_host, oref, osrc, Ps, [O.grey(im) for im in ims], it)
        seen = oref >= 0
        assert np.allclose(g["rho"][seen], o["rho"][seen], rtol=1e-12, atol=0)
        assert np.array_equal(np.isnan(g["sk"]), np.isnan(o["sk"]))
        ok = ~np.isnan(o["sk"])
        assert (np.abs(g["sk"][ok] - o["sk"][ok]) <= o["bound"][ok]).all()
        # k* agrees wherever the oracle's margin over the runner-up exceeds twice its bound
        for u in np.nonzero(seen & (o["kstar"] != O.NO_K))[0]:
            s = o["sk"][u]
            others = np.delete(s, o["kstar"][u] + O.K)
            margin = o["best"][u] - np.nanmax(others) if (~np.isnan(others)).any() else np.inf
            if not np.isnan(s[O.K]):          # the MIN_GAIN test is a decision too
                margin = min(margin, abs(np.nanmax(s) - s[O.K] - O.MIN_GAIN))
            if margin > 2 * o["bound"][u].max():
                assert g["kstar"][u] == o["kstar"][u]
                assert abs(g["d0"][u] - o["d0"][u]) <= 1e-9 * o["rho"][u]
                assert abs(g["conf"][u] - o["conf"][u]) <= o["bound"][u].max()
                checked_k += 1
        assert (g["kstar"][~seen] == O.NO_K).all() and (g["conf"][~seen] == 0).all()
        d = refine.smooth(nb, sw["d0"], sw["conf"])
        od = O.smooth(f, g["d0"], g["conf"])
        dh = d.cpu().numpy()
        assert np.abs(dh - od).max() <= 1e-12 * max(np.abs(g["d0"]).max(), 1e-30)
        cur = refine.apply(cur, normal, d)
        assert np.array_equal(cur.cpu().numpy(), O.apply(host, n_host, dh))
        host = cur.cpu().numpy()
    assert checked_k > 0.7 * V


def _refine(v, c, f, ims, Ps, srcs, **kw):
    out = refine.refine_mesh(_cuda(v), _cuda(c), _cuda(f), [_cuda(im) for im in ims], Ps, srcs,
                             log=lambda *a: None, **kw)
    return out


@pytest.mark.parametrize("name", sorted(SCENES))
def test_whole_call_agrees_with_the_oracle_and_repeats_bit_for_bit(name):
    ims, Ps, srcs = _views(name)
    v, c, f = _bumpy()
    V1, C1, F1, st = _refine(v, c, f, ims, Ps, srcs)
    V2, C2, F2, _ = _refine(v, c, f, ims, Ps, srcs)
    assert torch.equal(V1, V2) and torch.equal(C1, C2) and torch.equal(F1, F2)
    assert np.array_equal(C1.cpu().numpy(), c) and np.array_equal(F1.cpu().numpy(), f)
    assert V1.dtype == torch.float32 and V1.shape == v.shape
    o = O.refine_mesh(v, f, ims, Ps, srcs, 3)
    rho = np.median(o["iterations"][0]["rho"][o["iterations"][0]["ref"] >= 0])
    err = np.linalg.norm(V1.cpu().numpy().astype(np.float64) - o["verts"], axis=1)
    # a vertex whose k* sits within rounding of a tie may take the other k in one iteration and
    # then carry that difference; every other vertex agrees to rounding
    assert (err <= 1e-6 * rho).mean() >= 0.99 and err.max() <= 2 * rho
    assert len(st["per_iteration"]) == 3
    for s, it in zip(st["per_iteration"], o["iterations"]):
        assert abs(s["seen"] - (it["ref"] >= 0).sum()) <= 2
        assert abs(s["confident"] - (it["conf"] > 0).sum()) <= 2
        assert 0.3 <= s["mean_score"] <= 1 and s["mean_move"] >= 0
    moved = np.linalg.norm(V1.cpu().numpy() - v, axis=1)
    assert (moved > 0).mean() > 0.7 and moved[-1] == 0            # the unused vertex stays


def test_refinement_pulls_a_lifted_mesh_onto_the_plane():
    ims, Ps, srcs = O.plane_scene()
    v, c, f = _bumpy()
    before = np.sqrt(np.mean(v[:-1, 2].astype(np.float64) ** 2))
    V1, _, _, _ = _refine(v, c, f, ims, Ps, srcs)
    z = V1.cpu().numpy()[:-1, 2].astype(np.float64)
    assert np.sqrt(np.mean(z ** 2)) < 0.4 * before


def test_a_textureless_scene_leaves_the_vertices_bit_identical():
    ims, Ps, srcs = O.plane_scene(constant=(90, 140, 200))
    v, c, f = _bumpy()
    V1, C1, F1, st = _refine(v, c, f, ims, Ps, srcs)
    assert np.array_equal(V1.cpu().numpy(), v)
    assert st["per_iteration"][0]["seen"] > 0
    assert all(s["confident"] == 0 for s in st["per_iteration"])


def test_bad_inputs_and_oversized_work_are_refused():
    ims, Ps, srcs = O.plane_scene()
    v, c, f = _bumpy()
    bad = f.copy()
    bad[3, 1] = len(v)
    with pytest.raises(ValueError, match="index outside"):
        _refine(v, c, bad, ims, Ps, srcs)
    with pytest.raises(ValueError, match="source 5"):
        _refine(v, c, f, ims, Ps, [[1, 2], [5], [], [], []])
    with pytest.raises(ValueError, match="source lists"):
        _refine(v, c, f, ims, Ps, srcs[:4])
    for it in (0, -1, 1.5, True):
        with pytest.raises(ValueError, match="iterations"):
            _refine(v, c, f, ims, Ps, srcs, iterations=it)
    with pytest.raises(_lib.CasMVSError, match="bytes"):
        _refine(v, c, f, ims, Ps, srcs, max_bytes=1000)


def test_the_command_line_writes_what_the_function_returns(tmp_path):
    ims, Ps, srcs = O.plane_scene()
    v, c, f = _bumpy()
    from PIL import Image
    from casmvsnet_pl_b200 import mesh
    (tmp_path / "cams").mkdir()
    (tmp_path / "images").mkdir()
    for j, (im, P) in enumerate(zip(ims, Ps)):
        # the camera file holds E = P and K = I: the same world -> pixel matrix
        with open(tmp_path / "cams" / f"{j:08d}_cam.txt", "w") as fh:
            fh.write("extrinsic\n" + "\n".join(" ".join(f"{x:.9g}" for x in row)
                                                for row in P.astype(np.float64)) +
                     "\n\nintrinsic\n1 0 0\n0 1 0\n0 0 1\n\n1 1\n")
        Image.fromarray(im).save(tmp_path / "images" / f"{j:08d}.png")
    with open(tmp_path / "pair.txt", "w") as fh:
        fh.write(f"{len(ims)}\n" + "".join(f"{j}\n{len(s)} " + " ".join(f"{x} 1" for x in s) + "\n"
                                          for j, s in enumerate(srcs)))
    mesh.write_mesh_ply(tmp_path / "in.ply", v, c, f)
    refine.main(["--ply", str(tmp_path / "in.ply"), "--cams", str(tmp_path / "cams"), "--images",
                 str(tmp_path / "images"), "--pair", str(tmp_path / "pair.txt"), "--iterations", "2",
                 "--out", str(tmp_path / "out.ply")])
    V2, C2, F2 = io.read_mesh_ply(tmp_path / "out.ply")
    V1, _, _, _ = _refine(v, c, f, ims, Ps, srcs, iterations=2)
    assert np.array_equal(V2, V1.cpu().numpy()) and np.array_equal(C2, c) and np.array_equal(F2, f)


def _tree_bytes(d):
    return {os.path.relpath(os.path.join(r, n), d): open(os.path.join(r, n), "rb").read()
            for r, _, files in os.walk(d) for n in files}


def test_eval_pipeline_mesh_refine_changes_only_the_mesh_vertices(tmp_path):
    from casmvsnet_pl_b200 import ABN, synth
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    root = tmp_path / "capture"
    synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), n_points=3000, seed=7,
                             textured=True)
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN)
    synth.randomize_model_(model, 0)
    ckpt = tmp_path / "weights.pt"
    torch.save(model.state_dict(), ckpt)
    common = ["--dataset_name", "colmap", "--root_dir", str(root), "--img_wh", "128", "96",
              "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0", "--ckpt", str(ckpt),
              "--mesh"]
    ep.main(common + ["--out", str(tmp_path / "plain")])
    ep.main(common + ["--mesh_refine", "--mesh_refine_iterations", "2", "--out",
                      str(tmp_path / "ref")])
    plain, ref = _tree_bytes(tmp_path / "plain"), _tree_bytes(tmp_path / "ref")
    ply = os.path.join("mesh", "capture.ply")
    assert sorted(plain) == sorted(ref)
    assert {k: b for k, b in ref.items() if k != ply} == {k: b for k, b in plain.items() if k != ply}
    assert any(k.startswith("depth") for k in plain) and os.path.join("points", "capture.ply") in plain
    v0, c0, f0 = io.read_mesh_ply(tmp_path / "plain" / ply)
    v1, c1, f1 = io.read_mesh_ply(tmp_path / "ref" / ply)
    assert np.array_equal(f0, f1) and np.array_equal(c0, c1) and len(f0) > 0
    assert v0.shape == v1.shape and not np.array_equal(v0, v1)
