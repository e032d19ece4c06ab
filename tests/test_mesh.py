"""Meshing without a GPU: the generated marching-cubes case table (closure, edge use, orientation,
the committed header in sync), the float64 extraction oracle on analytic signed-distance grids
(sphere, torus, two spheres meeting at an ambiguous face, random sign fields), the mesh PLY round
trip and the --mesh command line."""
import numpy as np
import pytest

from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import io as cio
from casmvsnet_pl_b200 import mc_table
from oracle import mesh_oracle as O


def _crossing_edges(case):
    return {e for e, (a, b) in enumerate(mc_table.EDGES) if ((case >> a) & 1) != ((case >> b) & 1)}


@pytest.mark.parametrize("case", range(256))
def test_case_loops_close_and_use_every_crossing_edge_once(case):
    loops = mc_table.case_loops(case)
    used = [e for loop in loops for e in loop]
    assert sorted(used) == sorted(_crossing_edges(case))            # each crossing edge once
    segs = set(mc_table.face_segments(case))
    for loop in loops:
        assert len(loop) >= 3
        for i, e in enumerate(loop):                                # consecutive = one segment
            assert (e, loop[(i + 1) % len(loop)]) in segs
    tris = mc_table.case_triangles(case)
    assert len(tris) == sum(len(loop) - 2 for loop in loops)
    for t in tris:
        assert set(t) <= _crossing_edges(case) and len(set(t)) == 3


def test_table_arrays_match_the_rule():
    tris, count, mask = mc_table.table()
    assert tris.shape == (256, int(count.max()), 3)
    for c in range(256):
        assert count[c] == len(mc_table.case_triangles(c))
        assert mask[c] == sum(1 << e for e in _crossing_edges(c))
        assert (tris[c, count[c]:] == -1).all()
    assert count[0] == 0 and count[255] == 0


def test_committed_header_equals_generator_output():
    with open(mc_table.HEADER) as f:
        assert f.read() == mc_table.header_text(), "run python -m casmvsnet_pl_b200.mc_table"


def _normal(tri):
    p = [mc_table._mid(e) for e in tri]
    return np.cross(p[1] - p[0], p[2] - p[0])


@pytest.mark.parametrize("axis", range(3))
def test_half_space_cases_point_their_normals_out_of_the_inside(axis):
    """Corners with coordinate `axis` = 0 inside: every triangle's normal points to +axis; the
    complement points to -axis."""
    low = sum(1 << c for c in range(8) if not (c >> axis) & 1)
    for case, sign in ((low, 1.0), (255 ^ low, -1.0)):
        tris = mc_table.case_triangles(case)
        assert tris
        for t in tris:
            n = _normal(t)
            assert sign * n[axis] > 0 and np.allclose(np.delete(n, axis), 0)


@pytest.mark.parametrize("corner", range(8))
def test_single_corner_cases_point_away_from_the_corner(corner):
    for case, sign in ((1 << corner, 1.0), (255 ^ (1 << corner), -1.0)):
        (t,) = mc_table.case_triangles(case)
        centre = np.mean([mc_table._mid(e) for e in t], axis=0)
        assert sign * np.dot(_normal(t), centre - mc_table.corner_pos(corner)) > 0


def _grid(f, n, off):
    i = np.arange(n, dtype=np.float64) + off
    return f(*np.meshgrid(i, i, i, indexing="ij"))


def _mesh(sdf, origin):
    keys, tsdf, weight, color = O.grid_volume(sdf, origin)
    return O.extract(keys, tsdf, weight, color, 1.0)


def test_sphere_is_closed_oriented_genus_zero_and_accurate():
    r, c = 20.0, np.array([0.3, -0.2, 0.1])
    v, col, f = _mesh(_grid(lambda x, y, z: np.sqrt((x - c[0])**2 + (y - c[1])**2 + (z - c[2])**2) - r,
                            48, -24), (-24, -24, -24))
    assert O.is_closed_oriented(f)
    assert O.euler_characteristic(len(v), f) == 2
    assert abs(O.signed_volume(v, f) / (4 / 3 * np.pi * r**3) - 1) < 0.01
    assert np.abs(np.linalg.norm(v - c, axis=1) - r).max() < 0.05
    assert (col == 128).all() and len(np.unique(f)) == len(v)        # every vertex used


def test_torus_has_euler_characteristic_zero():
    R, r = 16.0, 6.0
    v, _, f = _mesh(_grid(lambda x, y, z: np.sqrt((np.sqrt(x**2 + y**2) - R)**2 + z**2) - r, 52, -26),
                    (-26, -26, -26))
    assert O.is_closed_oriented(f)
    assert O.euler_characteristic(len(v), f) == 0
    assert abs(O.signed_volume(v, f) / (2 * np.pi**2 * R * r**2) - 1) < 0.01


def test_two_spheres_sharing_an_ambiguous_face_have_no_hole():
    """Spheres of radius 0.6 around voxels (5,5,5) and (6,6,5): the face z = 5 of the cells between
    them has its diagonal corners inside, the others outside."""
    sdf = _grid(lambda x, y, z: np.minimum(np.sqrt((x - 5)**2 + (y - 5)**2 + (z - 5)**2),
                                           np.sqrt((x - 6)**2 + (y - 6)**2 + (z - 5)**2)) - 0.6, 12, 0)
    assert sdf[5, 5, 5] < 0 and sdf[6, 6, 5] < 0 and sdf[6, 5, 5] > 0 and sdf[5, 6, 5] > 0
    v, _, f = _mesh(sdf, (0, 0, 0))
    assert O.is_closed_oriented(f)
    assert O.euler_characteristic(len(v), f) == 4                      # two spheres


@pytest.mark.parametrize("seed", range(4))
def test_random_sign_fields_give_closed_oriented_meshes(seed):
    """Any field that is positive on the grid border meshes into closed surfaces: every shared
    face is cut the same way from both sides (ambiguous faces included) and the orientations of
    neighbouring cells agree.  The grid straddles brick borders and negative brick coordinates."""
    rng = np.random.default_rng(seed)
    sdf = rng.choice([-1.0, 1.0], size=(14, 14, 14)) * rng.uniform(0.2, 1.0, (14, 14, 14))
    sdf[[0, -1]] = sdf[:, [0, -1]] = sdf[:, :, [0, -1]] = 1.0
    v, _, f = _mesh(sdf, (3, -5, 7))
    assert len(f) > 1000 and O.is_closed_oriented(f)


def test_mesh_ply_round_trip_and_point_reader(tmp_path):
    from casmvsnet_pl_b200 import mesh
    rng = np.random.default_rng(0)
    v = rng.normal(size=(50, 3)).astype(np.float32)
    c = rng.integers(0, 256, (50, 3)).astype(np.uint8)
    f = rng.integers(0, 50, (70, 3)).astype(np.int32)
    p = tmp_path / "m.ply"
    mesh.write_mesh_ply(str(p), v, c, f)
    v2, c2, f2 = cio.read_mesh_ply(str(p))
    assert v2.dtype == np.float32 and c2.dtype == np.uint8 and f2.dtype == np.int32
    assert np.array_equal(v, v2) and np.array_equal(c, c2) and np.array_equal(f, f2)
    pts = cio.read_ply(str(p))                       # the point reader reads the vertices only
    assert np.array_equal(np.stack([pts["x"], pts["y"], pts["z"]], 1), v)
    mesh.write_mesh_ply(str(p), v[:0], c[:0], f[:0])
    v3, c3, f3 = cio.read_mesh_ply(str(p))
    assert v3.shape == (0, 3) and c3.shape == (0, 3) and f3.shape == (0, 3)


def test_read_mesh_ply_rejects_point_clouds(tmp_path):
    from casmvsnet_pl_b200 import fusion
    p = tmp_path / "pts.ply"
    fusion.write_ply(str(p), np.zeros((3, 3), np.float32), np.zeros((3, 3), np.uint8))
    with pytest.raises(ValueError):
        cio.read_mesh_ply(str(p))


def test_mesh_arguments():
    a = ep.parse_args(["--root_dir", "x", "--dataset_name", "colmap"])
    assert a.mesh is False and a.mesh_voxel is None
    a = ep.parse_args(["--root_dir", "x", "--mesh"])
    assert a.mesh is True and a.mesh_voxel is None
    a = ep.parse_args(["--root_dir", "x", "--mesh", "--mesh_voxel", "0.25"])
    assert a.mesh and a.mesh_voxel == 0.25
    with pytest.raises(SystemExit):
        ep.parse_args(["--root_dir", "x", "--mesh", "--mesh_voxel", "0"])


def test_default_voxel_size_is_twice_the_median_footprint():
    import torch
    from casmvsnet_pl_b200 import mesh
    K = np.array([[100.0, 0, 32], [0, 100.0, 24], [0, 0, 1]])
    depths, Ps = [], []
    for z in (2.0, 4.0, 8.0):
        d = torch.zeros(48, 64)
        d[10:30, 10:40] = z
        P = np.eye(4)
        P[:3, :3] = K
        depths.append(d)
        Ps.append(P.astype(np.float32))
    depths.append(torch.zeros(48, 64))               # a view without depth does not count
    Ps.append(Ps[0])
    # footprint at depth z with focal 100: z / 100; median over (2, 4, 8) = 4 -> 2 * 0.04
    assert mesh.default_voxel_size(depths, Ps) == pytest.approx(0.08, rel=1e-6)
