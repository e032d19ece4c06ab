"""Mesh cleaning's rule on the numpy restatement (oracle/mesh_clean_oracle.py): holes closed on a
sphere, a square hole in a grid filled flat with its own area, the area guard, figure-eights and
taken diagonals skipped, the piece thresholds at their edges, and every flag refusal."""
import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import mesh_clean
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import mesh_clean_oracle as O
from oracle import mesh_oracle as M
from oracle import simplify_oracle as S


# ------------------------------------------------------------------------------ test meshes
def grid_without(n, cells):
    """S.grid_mesh(n) without the two faces of each cell (x, y) in `cells` -> (verts, faces)."""
    v, f = S.grid_mesh(n)
    drop = np.zeros(len(f), bool)
    for x, y in cells:
        c = y * n + x
        drop[c] = drop[n * n + c] = True
    return v, f[~drop]


def square_hole_grid(n=100, x0=40, y0=40, side=4):
    return grid_without(n, [(x, y) for x in range(x0, x0 + side) for y in range(y0, y0 + side)])


def sphere_with_fans_removed(grid=24, count=3):
    """S.sphere_mesh(grid) without the faces around `count` far-apart vertices."""
    v, c, f = S.sphere_mesh(grid)
    picks = []
    for axis in np.eye(3)[:count]:
        picks.append(int(np.argmax(v.astype(np.float64) @ axis)))
    drop = np.isin(f, picks).any(1)
    return v, c, f[~drop], picks


def pieces_mesh():
    """Three disjoint grids of 200, 50 and 2 faces, the small ones placed off to the side."""
    vs, fs, off = [], [], 0
    for n, dx in ((10, 0.0), (5, 3.0), (1, 6.0)):
        v, f = S.grid_mesh(n)
        v = v + np.array([dx, 0, 0], np.float32)
        vs.append(v)
        fs.append(f + off)
        off += len(v)
    v = np.concatenate(vs)
    return v, np.zeros_like(v, np.uint8), np.concatenate(fs).astype(np.int32)


def pillow(a, b, apex):
    """Two faces on the same three vertices with opposite windings: a closed two-face piece that
    makes a -- b an interior edge."""
    return [[a, b, apex], [b, a, apex]]


def quad_hole_with_taken_diagonals():
    """A 4 x 4 grid without its middle-left cell, whose two diagonals are both edges of closed
    pillows elsewhere."""
    n = 4
    v, f = grid_without(n, [(1, 1)])
    a, b, c, d = 1 * 5 + 1, 1 * 5 + 2, 2 * 5 + 2, 2 * 5 + 1
    extra_v = np.array([[0.3, 0.3, 1.0], [0.4, 0.3, 1.0]], np.float32)
    e1, e2 = len(v), len(v) + 1
    f = np.concatenate([f, pillow(a, c, e1), pillow(b, d, e2)]).astype(np.int32)
    v = np.concatenate([v, extra_v])
    return v, np.zeros_like(v, np.uint8), f


def figure_eight_grid():
    """A 20 x 20 grid without two 2 x 2 blocks that touch at one vertex."""
    cells = [(x, y) for x in (6, 7) for y in (6, 7)] + [(x, y) for x in (8, 9) for y in (8, 9)]
    return grid_without(20, cells)


def directed_edge_counts(faces):
    f = np.asarray(faces, np.int64)
    g = np.roll(f, -1, 1)
    d = (f << 32 | g).ravel()
    return np.unique(d, return_counts=True)


def _colours(v):
    return np.zeros((len(v), 3), np.uint8)


# ------------------------------------------------------------------------------ holes
def test_a_sphere_with_three_fans_removed_comes_back_closed():
    v, c, f, picks = sphere_with_fans_removed()
    assert not M.is_closed_oriented(f)
    V, C, F, st = O.clean_mesh(v, c, f, max_hole=16)
    assert st["holes_filled"] == 3 and st["loops"] == 3 and st["loops_not_simple"] == 0
    assert M.is_closed_oriented(F) and M.euler_characteristic(len(V), F) == 2
    assert st["vertices"] == len(v) - 3 and st["faces"] == len(f) + st["faces_added"]
    assert M.signed_volume(V, F) > 0


def test_a_square_hole_in_a_grid_is_filled_flat_with_its_area():
    v, f = square_hole_grid()
    V, C, F, st = O.clean_mesh(v, _colours(v), f, max_hole=16)
    assert st["loops"] == 2 and st["holes_filled"] == 1 and st["holes_too_large"] == 1
    assert st["faces_added"] == 14                       # 16 boundary vertices, no interior one
    fill = F[len(f):]
    p = V.astype(np.float64)[fill]
    assert np.abs(p[:, :, 2]).max() == 0                 # in the plane
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    assert (np.linalg.norm(n, axis=1) > 0).all()         # no zero-area face on the collinear sides
    assert (n[:, 2] > 0).all()                           # the grid's own winding
    area = 0.5 * np.linalg.norm(n, axis=1).sum()
    assert area == pytest.approx(16 * 0.01 ** 2, rel=1e-6)
    # every edge of the hole now has two faces; the outer border of 400 edges is still open
    _, uc, _, dc = M.edge_counts(F)
    assert (dc == 1).all() and (uc == 1).sum() == 400


def test_a_surviving_disc_is_not_capped():
    v, f = S.grid_mesh(4)
    V, C, F, st = O.clean_mesh(v, _colours(v), f, max_hole=16)
    assert st["loops"] == 1 and st["holes_area_guard"] == 1 and st["holes_filled"] == 0
    assert np.array_equal(F, f) and np.array_equal(V, v)
    v1 = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    V, C, F, st = O.clean_mesh(v1, _colours(v1), np.array([[0, 1, 2]]), max_hole=3)
    assert st["holes_area_guard"] == 1 and len(F) == 1


def test_a_figure_eight_loop_is_skipped_and_counted():
    v, f = figure_eight_grid()
    V, C, F, st = O.clean_mesh(v, _colours(v), f, max_hole=16)
    assert st["loops_not_simple"] == 2 and st["holes_filled"] == 0
    assert st["loops"] == 1 and st["holes_too_large"] == 1      # the outer border
    assert len(F) == len(f)


def test_a_hole_whose_triangulations_all_use_an_existing_edge_is_skipped():
    v, c, f = quad_hole_with_taken_diagonals()
    V, C, F, st = O.clean_mesh(v, c, f, min_ratio=0, max_hole=8)
    assert st["holes_no_triangulation"] == 1 and st["holes_filled"] == 0
    assert st["holes_too_large"] == 1 and st["pieces"] == 3 and len(F) == len(f)
    # without the pillows the hole is filled with two triangles
    V, C, F, st = O.clean_mesh(v, c, f[:-4], min_ratio=0, max_hole=8)
    assert st["holes_filled"] == 1 and st["faces_added"] == 2


def test_a_closed_piece_is_untouched():
    v, c, f = S.sphere_mesh(16)
    V, C, F, st = O.clean_mesh(v, c, f, max_hole=128)
    assert st["loops"] == 0 and st["loops_not_simple"] == 0 and st["faces_added"] == 0
    assert np.array_equal(F, f) and np.array_equal(V, v) and np.array_equal(C, c)


def test_fill_faces_meet_every_boundary_half_edge_reversed():
    v, c, f, _ = sphere_with_fans_removed()
    V, C, F, st = O.clean_mesh(v, c, f, max_hole=16)
    d, n = directed_edge_counts(F)
    assert (n == 1).all()


# ------------------------------------------------------------------------------ pieces
@pytest.mark.parametrize("kw, kept", [
    (dict(min_ratio=0), [200, 50, 2]),
    (dict(min_ratio=1), [200]),
    (dict(min_ratio=0, min_faces=50), [200, 50]),
    (dict(min_ratio=0, min_faces=51), [200]),
    (dict(min_ratio=0.25), [200, 50]),              # ceil(0.25 x 200) = 50, exactly the piece
    (dict(min_ratio=0.01), [200, 50, 2]),           # ceil(2.0) = 2
    (dict(min_ratio=0.0101), [200, 50]),            # ceil(2.02) = 3
])
def test_piece_thresholds_at_their_edges(kw, kept):
    v, c, f = pieces_mesh()
    V, C, F, st = O.clean_mesh(v, c, f, **kw)
    assert st["pieces"] == 3 and st["pieces_removed"] == 3 - len(kept)
    assert len(F) == sum(kept) and st["faces_removed"] == 252 - sum(kept)
    assert st["vertices"] == {200: 121, 50: 36, 2: 4}[200] + sum({50: 36, 2: 4}[k] for k in kept[1:])


def test_degenerate_faces_are_dropped_and_counted():
    v, f = S.grid_mesh(3)
    f = np.concatenate([f, [[0, 0, 1], [0, 1, 2]]]).astype(np.int32)    # repeated, collinear
    V, C, F, st = O.clean_mesh(v, _colours(v), f)
    assert st["degenerate"] == 2 and len(F) == 18


def test_piece_areas_sum_in_face_order_by_chunks():
    v, f = S.grid_mesh(40)                                 # 3200 faces: chunks of 1024, 1024, 1024, 128
    v2, f2 = S.grid_mesh(2)
    f = np.concatenate([f[:1500], f2 + len(v), f[1500:]]).astype(np.int32)
    v = np.concatenate([v, v2 + np.float32(5)])
    pc = O.pieces(v, f)
    assert list(pc["count"]) == [3200, 8]
    a = O.face_area(v, f)
    big = np.concatenate([a[:1500], a[1508:]])
    sums = []
    for k in range(0, 3200, 1024):
        s = 0.0
        for x in big[k:k + 1024]:
            s = s + x
        sums.append(s)
    s = 0.0
    for x in sums:
        s = s + x
    assert pc["area"][0] == s
    s = 0.0
    for x in a[1500:1508]:
        s = s + x
    assert pc["area"][1] == s


# ------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("kw, msg", [
    (dict(min_faces=-1), "min_faces"),
    (dict(min_faces=1.5), "min_faces"),
    (dict(min_ratio=-0.1), "min_ratio"),
    (dict(min_ratio=1.5), "min_ratio"),
    (dict(min_ratio=float("nan")), "min_ratio"),
    (dict(max_hole=2), "max_hole"),
    (dict(max_hole=129), "max_hole"),
    (dict(max_hole=-3), "max_hole"),
])
def test_bad_options_are_refused_before_anything_runs(kw, msg):
    v = torch.zeros(3, 3)
    with pytest.raises(ValueError, match=msg):
        mesh_clean.clean_mesh(v, torch.zeros(3, 3, dtype=torch.uint8),
                              torch.tensor([[0, 1, 2]]), **kw)


def test_cpu_tensors_are_refused():
    with pytest.raises(ValueError, match="CUDA tensor"):
        mesh_clean.clean_mesh(torch.zeros(3, 3), torch.zeros(3, 3, dtype=torch.uint8),
                              torch.tensor([[0, 1, 2]]))


@pytest.mark.parametrize("argv, msg", [
    (["--min_faces", "-1"], "--min_faces"),
    (["--min_ratio", "1.5"], "--min_ratio"),
    (["--min_ratio", "nan"], "--min_ratio"),
    (["--max_hole", "2"], "--max_hole"),
    (["--max_hole", "129"], "--max_hole"),
])
def test_cli_flag_refusals(argv, msg, capsys):
    with pytest.raises(SystemExit):
        mesh_clean.parse_args(["--ply", "a.ply", "--out", "b.ply"] + argv)
    assert msg in capsys.readouterr().err


def test_cli_defaults():
    a = mesh_clean.parse_args(["--ply", "a.ply", "--out", "b.ply"])
    assert (a.min_faces, a.min_ratio, a.max_hole) == (0, 0.01, 0)


@pytest.mark.parametrize("extra, msg", [
    (["--mesh_clean"], "--mesh_clean needs --mesh"),
    (["--mesh", "--mesh_clean_ratio", "0.1"], "--mesh_clean_ratio needs --mesh_clean"),
    (["--mesh", "--mesh_max_hole", "8"], "--mesh_max_hole needs --mesh_clean"),
    (["--mesh", "--mesh_clean", "--mesh_clean_ratio", "2"], "--mesh_clean_ratio must be"),
    (["--mesh", "--mesh_clean", "--mesh_max_hole", "1"], "--mesh_max_hole must be"),
    (["--mesh", "--mesh_clean", "--mesh_max_hole", "200"], "--mesh_max_hole must be"),
])
def test_eval_pipeline_flag_refusals(extra, msg, capsys):
    with pytest.raises(SystemExit):
        ep.parse_args(["--root_dir", "x"] + extra)
    assert msg in capsys.readouterr().err


def test_eval_pipeline_clean_options():
    assert ep._clean_options(ep.parse_args(["--root_dir", "x", "--mesh"])) is None
    a = ep.parse_args(["--root_dir", "x", "--mesh", "--mesh_clean"])
    assert ep._clean_options(a) == {}
    a = ep.parse_args(["--root_dir", "x", "--mesh", "--mesh_clean", "--mesh_clean_ratio", "0.05",
                       "--mesh_max_hole", "32"])
    assert ep._clean_options(a) == dict(min_ratio=0.05, max_hole=32)
