"""Seam levelling rules on the CPU (oracle/texture_level_oracle.py and the host code of texture.py):
two quads seen in two constant-colour views meet in the middle, identical views give no offset,
flat charts and open or non-manifold edges add no terms, and the flag refusals."""
import numpy as np
import pytest

from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import render, texture
from oracle import texture_level_oracle as L
from oracle import texture_oracle as T

WH = (64, 48)


def _view():
    """A camera at (0, 0, -5) looking down +z, f = 60, principal point at the image centre."""
    K = np.array([[60.0, 0, 31.5], [0, 60.0, 23.5], [0, 0, 1]])
    E = np.eye(4)
    E[:3, 3] = [0.0, 0.0, 5.0]
    return render.projection(K, E).astype(np.float32)


def _textured(verts, faces, labels, Ps, images, colours=None):
    """texture_oracle's steps 4-8 on given labels -> what the levelling takes."""
    verts = np.asarray(verts, np.float32)
    faces = np.asarray(faces, np.int64)
    labels = np.asarray(labels, np.int32)
    colours = np.zeros((len(verts), 3), np.uint8) if colours is None else colours
    nbr = T.neighbours(faces)
    comp = T.components(nbr, labels)
    rect = T.rects(verts, faces, labels, comp, Ps)
    F = len(faces)
    roots = np.nonzero(comp == np.arange(F))[0]
    lab = labels[roots]
    box = np.where((lab < 0)[:, None], np.array([0, 0, T.FLAT - 1, T.FLAT - 1]), rect[roots])
    w, h = box[:, 2] - box[:, 0] + 1, box[:, 3] - box[:, 1] + 1
    S = T.PAGE_SIDE
    page_c, ox, oy, n_pages = T.pack(roots, w, h, S)
    charts = np.concatenate([roots[:, None], lab[:, None], box, page_c[:, None], ox[:, None],
                             oy[:, None]], 1).astype(np.int32)
    atlas = np.zeros((n_pages, S, S, 3), np.uint8)
    for c in charts:
        r, vi, x0, y0, x1, y1, pg, cx, cy = (int(a) for a in c)
        if vi < 0:
            atlas[pg, cy:cy + T.FLAT, cx:cx + T.FLAT] = (colours[faces[r]].astype(np.int64).sum(0) + 1) // 3
        else:
            atlas[pg, cy:cy + y1 - y0 + 1, cx:cx + x1 - x0 + 1] = images[vi][y0:y1 + 1, x0:x1 + 1]
    slot = np.searchsorted(roots, comp).astype(np.int32)
    return dict(verts=verts, faces=faces, labels=labels, slot=slot, charts=charts, Ps=Ps,
                images=images, nbr=nbr, atlas=atlas)


def _level(s, g=None):
    return L.level(s["verts"], s["faces"], s["labels"], s["slot"], s["charts"], s["Ps"], s["images"],
                   s["nbr"], s["atlas"], g=g)


# two unit quads side by side on z = 0, sharing the edge x = 0 (vertices 1 and 4)
QUADS_V = np.array([[-1, -0.5, 0], [0, -0.5, 0], [1, -0.5, 0], [-1, 0.5, 0], [0, 0.5, 0],
                    [1, 0.5, 0]], np.float32)
QUADS_F = np.array([[0, 1, 4], [0, 4, 3], [1, 2, 5], [1, 5, 4]], np.int64)


def _constant(c):
    return np.broadcast_to(np.array(c, np.uint8), (WH[1], WH[0], 3)).copy()


def test_two_constant_views_meet_half_way():
    c1, c2 = (100, 50, 200), (140, 30, 180)
    P = _view()
    s = _textured(QUADS_V, QUADS_F, [0, 0, 1, 1], [P, P], [_constant(c1), _constant(c2)])
    o = _level(s)
    assert len(o["unknowns"]) == 8 and len(o["pair_keys"]) == 2        # vertices 1 and 4
    assert len(o["rec_sub"]) == 2                                       # 1 seam edge x 2 ends
    assert np.array_equal(o["fpair"], np.tile(np.array(c1 + c2, np.float64), (2, 1)))
    half = (np.array(c2, np.float64) - np.array(c1)) / 2
    chart = o["unknowns"] >> 32
    a = chart == s["slot"][0]
    # EPS damps the mean offsets by 1 / (1 + EPS N / (2 m)) = 1 / (1 + 1e-4), N = 4, m = 2
    assert np.allclose(o["g"][a], half, atol=0.01) and np.allclose(o["g"][~a], -half, atol=0.01)
    assert o["seam_rms_before"] == pytest.approx(np.sqrt(np.mean((half * 2) ** 2)))
    assert o["seam_rms_after"] < 0.01
    # every owned texel of both charts becomes the same colour, the rest keep theirs
    own = o["owner"] != L.EMPTY
    assert own.sum() > 100
    assert (o["atlas"][own] == np.array([120, 40, 190], np.uint8)).all()
    assert np.array_equal(o["atlas"][~own], s["atlas"][~own])
    # the matrix: one seam entry per pair side, SMOOTH_WEIGHT on the chart edges, EPS on top
    n = len(o["unknowns"])
    A = np.zeros((n, n))
    rows = np.repeat(np.arange(n), np.diff(o["rowptr"]))
    A[rows, o["col"]] = o["val"]
    assert np.array_equal(A, A.T) and (np.linalg.eigvalsh(A) > 0).all()
    assert np.allclose(A.sum(1), L.EPS)
    assert sorted(set(o["val"][o["val"] < 0])) == [-L.SMOOTH_WEIGHT, -1.0]


def test_identical_views_give_no_offset():
    P = _view()
    y, x = np.mgrid[:WH[1], :WH[0]]
    img = np.stack([x * 3, y * 5, (x + y) * 2], -1).astype(np.uint8)
    s = _textured(QUADS_V, QUADS_F, [0, 0, 1, 1], [P, P], [img, img.copy()])
    o = _level(s)
    assert len(o["pair_keys"]) == 2
    assert np.array_equal(o["fpair"][:, :3], o["fpair"][:, 3:])
    assert not o["rhs"].any() and not o["g"].any()
    assert np.array_equal(o["atlas"], s["atlas"]) and o["seam_rms_before"] == 0.0


def test_flat_charts_and_open_or_non_manifold_edges_add_no_terms():
    P = _view()
    # the two quads, a third quad beside the second (flat), and a fan of three faces on one edge
    v = np.concatenate([QUADS_V, np.array([[2, -0.5, 0], [2, 0.5, 0]], np.float32),
                        np.array([[-1, -1.5, 0], [0, -1.5, 0], [-0.5, -1.5, 0.5], [-0.5, -1.5, -0.5],
                                  [-0.5, -1.0, 0]], np.float32)])
    f = np.concatenate([QUADS_F, np.array([[2, 6, 7], [2, 7, 5]]),
                        np.array([[8, 9, 12], [9, 8, 10], [8, 9, 11]])])
    labels = [0, 0, 1, 1, -1, -1, 0, 1, 1]
    c1, c2 = (100, 50, 200), (140, 30, 180)
    s = _textured(v, f, labels, [P, P], [_constant(c1), _constant(c2)])
    assert (s["nbr"][6:] == -1).all()                                  # the fan's edge is shared
    o = _level(s)
    # seams: only the quads' shared edge; the quad / flat edge (vertices 2 and 5) and the fan's
    # non-manifold edge between labels 0 and 1 (vertices 8 and 9) add nothing
    pv = np.unique(o["unknowns"][o["pair_keys"] >> 32] & 0xFFFFFFFF)
    assert list(pv) == [1, 4]
    assert o["corner"][4:6].min() == -1 and o["corner"][4:6].max() == -1
    assert not np.isin(np.array([6, 7]), o["unknowns"] & 0xFFFFFFFF).any()
    flat = s["charts"][s["charts"][:, 1] < 0]
    for c in flat:
        assert (o["owner"][c[6], c[8]:c[8] + 4, c[7]:c[7] + 4] == L.EMPTY).all()
        assert np.array_equal(o["atlas"][c[6], c[8]:c[8] + 4, c[7]:c[7] + 4],
                              s["atlas"][c[6], c[8]:c[8] + 4, c[7]:c[7] + 4])


def test_nearest_point_rule():
    u = np.array([[0.0, 4.0, 0.0]] * 4)
    v = np.array([[0.0, 0.0, 4.0]] * 4)
    d, l = L.nearest(u, v, np.array([1.0, -1.0, 3.0, 1.0]), np.array([1.0, 2.0, 3.0, -1.5]))
    assert d[0] == 0.0 and np.allclose(l[0], [0.5, 0.25, 0.25])
    assert d[1] == 1.0 and np.allclose(l[1], [0.5, 0.0, 0.5])       # onto edge 2 -> 0
    assert d[2] == pytest.approx(np.sqrt(2.0)) and np.allclose(l[2], [0.0, 0.5, 0.5])
    assert d[3] == 1.5 and np.allclose(l[3], [0.75, 0.25, 0.0])
    # the reverse winding gives the same answer
    d2, l2 = L.nearest(u[:, ::-1].copy(), v[:, ::-1].copy(), np.array([1.0, -1.0, 3.0, 1.0]),
                       np.array([1.0, 2.0, 3.0, -1.5]))
    assert np.array_equal(d2, d) and np.allclose(l2[:, ::-1], l)


def test_constants_agree_with_the_oracle():
    assert (texture.SEAM_SAMPLES, texture.SMOOTH_WEIGHT, texture.LEVEL_EPS, texture.REACH) == (
        L.SEAM_SAMPLES, L.SMOOTH_WEIGHT, L.EPS, L.REACH)
    assert texture.REACH >= np.sqrt(2.0)


def test_level_flags_are_refused_without_texturing():
    with pytest.raises(SystemExit):
        ep.parse_args(["--root_dir", "x", "--mesh", "--mesh_texture_level"])
    a = ep.parse_args(["--root_dir", "x", "--mesh", "--mesh_texture", "--mesh_texture_level"])
    assert a.mesh_texture_level
    assert not ep.parse_args(["--root_dir", "x", "--mesh", "--mesh_texture"]).mesh_texture_level
    a = texture.parse_args(["--ply", "a.ply", "--cams", "c", "--images", "i", "--out", "m.obj",
                            "--level"])
    assert a.level
