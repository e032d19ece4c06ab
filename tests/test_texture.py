"""Mesh texturing rules on the CPU (oracle/texture_oracle.py and the host code of texture.py):
occlusion and grazing angles remove candidates, the smoothing rule on a strip worked by hand,
charts across manifold edges only, packing, the OBJ round trip and the refusals."""
import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import render, texture
from oracle import texture_oracle as T

WH = (64, 48)


def _view(eye=(0.0, 0.0, -5.0)):
    """A camera at `eye` looking down +z, f = 60, principal point at the image centre."""
    K = np.array([[60.0, 0, 31.5], [0, 60.0, 23.5], [0, 0, 1]])
    E = np.eye(4)
    E[:3, 3] = -np.asarray(eye)
    return render.projection(K, E).astype(np.float32)


def _quad(z, s=0.5, x=0.0):
    v = np.array([[x - s, -s, z], [x + s, -s, z], [x + s, s, z], [x - s, s, z]], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int64)


def _mesh(*parts):
    vs, fs, n = [], [], 0
    for v, f in parts:
        vs.append(v)
        fs.append(f + n)
        n += len(v)
    return np.concatenate(vs), np.concatenate(fs)


# a wall far behind everything, so that the nearest pixel of a vertex on a silhouette is drawn
WALL = _quad(20.0, 40.0)


def test_a_face_hidden_behind_another_gets_no_candidate():
    v, f = _mesh(_quad(0.0, 0.6), _quad(1.0, 0.3), WALL)     # the second quad lies behind the first
    P = _view()
    zb = T.key_buffer(v, f, P, WH)
    m, s = T.view_candidates(v, f, P, WH, zb)
    assert m[:2].all() and not m[2:].any()
    assert (s[:2] > 0).all()
    v2, f2 = _mesh(_quad(1.0, 0.3), WALL)                     # alone it is seen
    m2, _ = T.view_candidates(v2, f2, P, WH, T.key_buffer(v2, f2, P, WH))
    assert m2[:2].all()


def test_a_face_at_a_grazing_angle_gets_no_candidate():
    # a quad tilted almost edge-on (|cos| about 0.05 < MIN_COS) beside a frontal one
    a = np.radians(87.0)
    tilt = np.array([[-0.4, -0.4 * np.cos(a), 0.4 * np.sin(a)], [0.4, -0.4 * np.cos(a), 0.4 * np.sin(a)],
                     [0.4, 0.4 * np.cos(a), -0.4 * np.sin(a)], [-0.4, 0.4 * np.cos(a), -0.4 * np.sin(a)]],
                    np.float32)
    v, f = _mesh((tilt, np.array([[0, 1, 2], [0, 2, 3]])), _quad(0.0, 0.3, x=1.2), WALL)
    P = _view()
    m, _ = T.view_candidates(v, f, P, WH, T.key_buffer(v, f, P, WH))
    assert not m[:2].any() and m[2:4].all()


def test_faces_near_the_border_are_not_candidates():
    v, f = _mesh(_quad(0.0, 0.6), WALL)
    P = _view()
    zb = T.key_buffer(v, f, P, WH)
    assert T.view_candidates(v, f, P, WH, zb)[0][:2].all()
    v2 = v.copy()
    v2[:4, 0] += np.float32(2.35)                             # crosses u = W - 1 - PAD
    assert not T.view_candidates(v2, f, P, WH, T.key_buffer(v2, f, P, WH))[0].any()


def _strip(n):
    """n faces in a strip: face i shares an edge with i - 1 and i + 1."""
    v = np.array([[i // 2, i % 2, 0] for i in range(n + 2)], np.float32)
    f = np.array([[i, i + 1, i + 2] for i in range(n)], np.int64)
    return v, f


def test_the_smoothing_rule_on_a_strip_by_hand():
    _, f = _strip(6)
    nbr = T.neighbours(f)
    assert nbr.tolist() == [[-1, 1, -1], [0, 2, -1], [1, 3, -1], [2, 4, -1], [3, 5, -1],
                            [4, -1, -1]]
    view = np.array([[0, 1, -1, -1], [1, -1, -1, -1], [0, 1, -1, -1], [1, 0, -1, -1],
                     [1, 0, -1, -1], [0, -1, -1, -1]], np.int32)
    score = np.array([[10, 6, 0, 0], [9, 0, 0, 0], [10, 4, 0, 0], [8, 5, 0, 0], [8, 3, 0, 0],
                      [7, 0, 0, 0]], np.float32)
    lab = view[:, 0].copy()                                   # 0 1 0 1 1 0
    r1 = T.smooth_round(nbr, score, view, lab)
    # face 0 has one neighbour: kept.  face 1: neighbours 0, 0 -> 0 is not its candidate: kept.
    # face 2: neighbours 1, 1 -> 1 scores 4 < 5: kept.  face 3: neighbours 0, 1 -> no pair: kept.
    # face 4: neighbours 1, 0: kept.  face 5: one neighbour: kept.
    assert r1.tolist() == [0, 1, 0, 1, 1, 0]
    score[2, 1] = 5                                           # now >= 0.5 x 10: face 2 takes 1
    r1 = T.smooth_round(nbr, score, view, lab)
    assert r1.tolist() == [0, 1, 1, 1, 1, 0]
    r2 = T.smooth_round(nbr, score, view, r1)                 # Jacobi: face 3 saw 1, 1 -> 1
    assert r2.tolist() == [0, 1, 1, 1, 1, 0]


def test_components_follow_equal_labels_across_manifold_edges_only():
    v, f = _strip(5)
    f = np.concatenate([f, [[2, 3, 7]]])                      # a third face on edge 2-3
    nbr = T.neighbours(f)
    assert (nbr[1] == -1).sum() == 2 and (nbr[2] == -1).sum() == 2       # 2-3 is non-manifold
    labels = np.array([4, 4, 4, 4, 2, 4], np.int32)
    comp = T.components(nbr, labels)
    assert comp.tolist() == [0, 0, 2, 2, 4, 5]                # no join across 1-2 (edge 2-3)
    labels = np.array([4, -1, 4, 4, 4, -1], np.int32)
    assert T.components(nbr, labels).tolist() == [0, 1, 2, 2, 2, 5]
    t = torch.from_numpy(f)
    assert np.array_equal(texture.neighbours(t).numpy(), nbr)


def test_packing_never_overlaps_stays_in_the_page_and_repeats():
    rng = np.random.default_rng(0)
    n = 3000
    w, h = rng.integers(4, 700, n), rng.integers(4, 700, n)
    ids = rng.permutation(10 * n)[:n]
    S = texture.page_side(w, h)
    assert S == 4096
    page, ox, oy, n_pages = texture.pack(ids, w, h, S)
    again = texture.pack(ids, w, h, S)
    assert all(np.array_equal(a, b) for a, b in zip((page, ox, oy), again[:3]))
    assert n_pages == again[3] == page.max() + 1
    assert all(np.array_equal(a, b) for a, b in zip((page, ox, oy), T.pack(ids, w, h, S)[:3]))
    assert (ox >= 0).all() and (oy >= 0).all() and (ox + w <= S).all() and (oy + h <= S).all()
    for p in range(n_pages):
        sel = np.nonzero(page == p)[0]
        occ = np.zeros((S, S), np.uint8)
        for i in sel:
            assert not occ[oy[i]:oy[i] + h[i], ox[i]:ox[i] + w[i]].any()
            occ[oy[i]:oy[i] + h[i], ox[i]:ox[i] + w[i]] = 1
    assert texture.page_side([5000], [10]) == 8192
    with pytest.raises(ValueError, match="does not fit"):
        texture.page_side([16385], [4])


def test_obj_mtl_png_round_trip(tmp_path):
    rng = np.random.default_rng(1)
    v = rng.standard_normal((50, 3)).astype(np.float32)
    f = rng.integers(0, 50, (40, 3)).astype(np.int32)
    uv = rng.random((40, 3, 2)).astype(np.float32)
    page = rng.integers(0, 3, 40).astype(np.int32)
    atlas = rng.integers(0, 256, (3, 16, 16, 3)).astype(np.uint8)
    out = texture.write_textured_obj(tmp_path / "m.obj", v, f, uv, page, atlas)
    assert [p.rsplit("/", 1)[-1] for p in out] == ["m.obj", "m.mtl", "m_0.png", "m_1.png", "m_2.png"]
    V, F, UV, PG, A = texture.read_textured_obj(tmp_path / "m.obj")
    assert np.array_equal(V.view(np.uint32), v.view(np.uint32))
    assert np.array_equal(F, f) and np.array_equal(PG, page) and np.array_equal(A, atlas)
    assert np.array_equal(UV.view(np.uint32), uv.view(np.uint32))
    text = (tmp_path / "m.obj").read_text().splitlines()
    used = [ln for ln in text if ln.startswith("usemtl")]
    assert used == ["usemtl page_0", "usemtl page_1", "usemtl page_2"]
    assert "map_Kd m_1.png" in (tmp_path / "m.mtl").read_text()


def test_texture_mesh_and_cli_refusals(tmp_path):
    v = torch.zeros(3, 3)
    with pytest.raises(ValueError, match="CUDA tensor"):
        texture.texture_mesh(v, torch.zeros(3, 3, dtype=torch.uint8), torch.zeros(1, 3, dtype=torch.int32),
                             [], [])
    with pytest.raises(SystemExit):
        texture.parse_args(["--ply", "a.ply", "--cams", "c", "--images", "i", "--out", "m.ply"])
    cams, imgs = tmp_path / "cams", tmp_path / "images"
    cams.mkdir()
    imgs.mkdir()
    with pytest.raises(ValueError, match="no \\*_cam.txt"):
        texture.read_views(str(cams), str(imgs))
    cam = "extrinsic\n1 0 0 0\n0 1 0 0\n0 0 1 0\n0 0 0 1\n\nintrinsic\n10 0 5\n0 10 5\n0 0 1\n\n1 1\n"
    for i in range(2):
        (cams / f"{i:08d}_cam.txt").write_text(cam)
    from PIL import Image
    Image.fromarray(np.zeros((8, 8, 3), np.uint8)).save(imgs / "a.png")
    with pytest.raises(ValueError, match="1 images and .* 2 cameras"):
        texture.read_views(str(cams), str(imgs))
    (tmp_path / "vn.txt").write_text("0 a.png\n")
    with pytest.raises(ValueError, match="no image name for view 1"):
        texture.read_views(str(cams), str(imgs), str(tmp_path / "vn.txt"))
    (tmp_path / "vn.txt").write_text("0 a.png\n1 b.png\n")
    paths, Ps = texture.read_views(str(cams), str(imgs), str(tmp_path / "vn.txt"))
    assert [p.rsplit("/", 1)[-1] for p in paths] == ["a.png", "b.png"] and Ps[0].shape == (4, 4)


def test_eval_pipeline_refuses_mesh_texture_without_mesh():
    with pytest.raises(SystemExit):
        ep.parse_args(["--root_dir", "x", "--mesh_texture"])
    a = ep.parse_args(["--root_dir", "x", "--mesh", "--mesh_texture"])
    assert a.mesh_texture and not ep.parse_args(["--root_dir", "x", "--mesh"]).mesh_texture


def test_render_refuses_textured_without_mesh():
    with pytest.raises(SystemExit):
        render.parse_args(["--dataset_name", "dtu", "--scan", "scan1", "--textured"])
