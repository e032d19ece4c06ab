"""Rendering without a GPU: Open3D viewpoint files (a hand-written fixture, the write / read round
trip, malformed files), the default view, known answers of the float32 restatement of the
kernels (pixel rule, depth test, point sizes, triangle coverage and depth) and the command line
with the renderer replaced by that restatement."""
import json
import math
import os

import numpy as np
import pytest

from casmvsnet_pl_b200 import fusion, mesh, render
from oracle import render_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "render")
EYE_P = np.eye(4, dtype=np.float32)           # u = X / Z, v = Y / Z, w = Z


# ---------------------------------------------------------------------------- viewpoint files
def test_open3d_fixture_reads_column_major():
    K, E, wh = render.read_camera(os.path.join(GOLDEN, "viewpoint.json"))
    assert wh == (640, 480)
    assert np.array_equal(K, [[500, 0, 300], [0, 520, 250], [0, 0, 1]])
    # a rotation by 90 degrees about z is not symmetric: row-major reading would transpose it
    assert np.array_equal(E, [[0, -1, 0, 1.5], [1, 0, 0, -2], [0, 0, 1, 3.25], [0, 0, 0, 1]])
    P, wh2 = render.read_viewpoint(os.path.join(GOLDEN, "viewpoint.json"))
    assert wh2 == wh and np.array_equal(P[:3], K @ E[:3]) and np.array_equal(P[3], [0, 0, 0, 1])
    # Open3D accepts back only fx == fy and the centred principal point: this K is refused
    with pytest.raises(ValueError, match="fx == fy"):
        render.write_viewpoint("unused.json", K, E, wh)


def test_write_then_read_round_trips_exactly(tmp_path):
    rng = np.random.default_rng(0)
    K, E = render.default_view(rng.normal(size=(100, 3)) * [3.0, 1.0, 0.2] + 0.1, (1280, 720))
    ang = 0.3
    R = np.array([[math.cos(ang), 0, math.sin(ang)], [0, 1, 0], [-math.sin(ang), 0, math.cos(ang)]])
    E[:3, :3] = R @ E[:3, :3]
    E[:3, 3] = [0.1234567890123, -7.0 / 3.0, 1e-17]
    path = str(tmp_path / "vp.json")
    render.write_viewpoint(path, K, E, (1280, 720))
    K2, E2, wh = render.read_camera(path)
    assert wh == (1280, 720) and np.array_equal(K2, K) and np.array_equal(E2, E)
    data = json.load(open(path))
    assert data["class_name"] == "PinholeCameraParameters"
    assert (data["version_major"], data["version_minor"]) == (1, 0)
    assert data["intrinsic"]["intrinsic_matrix"][6:8] == [639.5, 359.5]   # column-major cx, cy


def _mutate(data, key, value):
    d = json.loads(json.dumps(data))
    node, parts = d, key.split(".")
    for p in parts[:-1]:
        node = node[p]
    if value is KeyError:
        del node[parts[-1]]
    else:
        node[parts[-1]] = value
    return d


@pytest.mark.parametrize("key, value", [
    ("class_name", KeyError), ("class_name", "PinholeCameraIntrinsic"),
    ("version_major", 2), ("version_minor", KeyError),
    ("extrinsic", KeyError), ("extrinsic", [0.0] * 15), ("extrinsic", ["1"] * 16),
    ("extrinsic", [1.0] * 16),                                 # last row is not 0 0 0 1
    ("intrinsic", KeyError), ("intrinsic", [1, 2]),
    ("intrinsic.width", 0), ("intrinsic.height", 2.5), ("intrinsic.height", KeyError),
    ("intrinsic.intrinsic_matrix", [1.0] * 9), ("intrinsic.intrinsic_matrix", [1.0] * 8),
    ("intrinsic.intrinsic_matrix", KeyError),
])
def test_malformed_viewpoint_names_the_key(tmp_path, key, value):
    data = json.load(open(os.path.join(GOLDEN, "viewpoint.json")))
    path = tmp_path / "vp.json"
    path.write_text(json.dumps(_mutate(data, key, value)))
    with pytest.raises(ValueError, match=f"'{key}'"):
        render.read_camera(str(path))


def test_non_json_viewpoint_is_a_value_error(tmp_path):
    p = tmp_path / "vp.json"
    p.write_text("{not json")
    with pytest.raises(ValueError, match="not a JSON file"):
        render.read_camera(str(p))
    p.write_text("[1, 2]")
    with pytest.raises(ValueError, match="one JSON object"):
        render.read_camera(str(p))


# ---------------------------------------------------------------------------- default view
def _pixel(P, X):
    q = P @ np.append(X, 1.0)
    return q[:2] / q[2], q[2]


@pytest.mark.parametrize("lo, hi, wh", [
    ((-1, -2, -3), (4, 1, 0.5), (1920, 1080)),
    ((10, 10, 10), (10.5, 30, 11), (640, 480)),          # tall box: the y extent rules
    ((0, 0, 0), (200, 1, 1), (1280, 720)),               # flat wide box
])
def test_default_view_centres_the_box_and_keeps_its_corners_in_view(lo, hi, wh):
    lo, hi = np.array(lo, float), np.array(hi, float)
    corners = np.array([[(lo, hi)[i][0], (lo, hi)[j][1], (lo, hi)[k][2]]
                        for i in (0, 1) for j in (0, 1) for k in (0, 1)])
    pts = np.concatenate([corners, [[np.nan, 0, 0], [np.inf, 1, 1]]])     # non-finite ignored
    K, E = render.default_view(pts.astype(np.float32), wh)
    W, H = wh
    assert K[0, 0] == K[1, 1] == (H / 2) / math.tan(math.radians(30))
    assert (K[0, 2], K[1, 2]) == (W / 2 - 0.5, H / 2 - 0.5)
    assert np.allclose(E[:3, :3], [[1, 0, 0], [0, -1, 0], [0, 0, -1]])
    P = render.projection(K, E)
    uv, w = _pixel(P, (lo + hi) / 2)
    assert np.allclose(uv, (W / 2 - 0.5, H / 2 - 0.5), atol=1e-9) and w > 0
    # the distance is 0.7 max extent / tan 30 from the centre, along +z
    eye = -E[:3, :3].T @ E[:3, 3]
    assert np.allclose(eye, (lo + hi) / 2 + [0, 0, 0.7 * (hi - lo).max() / math.tan(math.radians(30))])
    for c in corners:
        uv, w = _pixel(P, c)
        assert w > 0 and -0.5 <= uv[0] < W - 0.5 and -0.5 <= uv[1] < H - 0.5, (c, uv)


def test_default_view_of_one_point_uses_unit_extent():
    K, E = render.default_view(np.array([[1.0, 2.0, 3.0]]), (100, 100))
    eye = -E[:3, :3].T @ E[:3, 3]
    assert np.allclose(eye, [1, 2, 3 + 0.7 / math.tan(math.radians(30))])
    assert np.allclose(render.camera_centre(render.projection(K, E)), eye, rtol=1e-6)


# ---------------------------------------------------------------------------- restatement: points
def _points(uvw):
    """Points that project to (u, v) at depth w under EYE_P."""
    uvw = np.asarray(uvw, np.float64)
    return np.stack([uvw[:, 0] * uvw[:, 2], uvw[:, 1] * uvw[:, 2], uvw[:, 2]], 1).astype(np.float32)


def _drawn(depth):
    return sorted(map(tuple, np.argwhere(depth > 0)[:, ::-1].tolist()))     # (x, y)


@pytest.mark.parametrize("u, px", [(2.0, 2), (2.5, 2), (np.nextafter(np.float32(2.5), np.float32(3)), 3),
                                   (1.5, 1), (2.49, 2), (-0.49, 0), (-0.5, None), (7.5, 7),
                                   (7.51, None)])
def test_a_point_lands_on_the_half_open_pixel(u, px):
    img, depth, _ = O.render_points(_points([[u, 3.0, 1.0]]), [[10, 20, 30]], EYE_P, (8, 6))
    assert _drawn(depth) == ([] if px is None else [(px, 3)])
    if px is not None:
        assert tuple(img[3, px]) == (10, 20, 30) and depth[3, px] == 1.0
    assert (img[depth == 0] == O.BACKGROUND).all()


def test_nearest_point_wins_and_a_tie_goes_to_the_lower_index():
    pts = _points([[1, 1, 2.0], [1, 1, 1.5], [1, 1, 3.0],     # nearest is index 1
                   [4, 2, 2.0], [4, 2, 2.0],                  # exact tie: index 3
                   [2, 4, 5.0], [2, 4, 5.0]])                 # the same point twice: index 5
    rgb = np.arange(21, dtype=np.uint8).reshape(7, 3)
    img, depth, zbuf = O.render_points(pts, rgb, EYE_P, (6, 6))
    assert tuple(img[1, 1]) == tuple(rgb[1]) and depth[1, 1] == 1.5
    assert tuple(img[2, 4]) == tuple(rgb[3]) and depth[2, 4] == 2.0
    assert tuple(img[4, 2]) == tuple(rgb[5])
    assert int(zbuf[4 * 6 + 2]) & 0xFFFFFFFF == 5
    # the key orders by depth first: reversing the list moves the tie to the other point
    img2, _, _ = O.render_points(pts[::-1].copy(), rgb[::-1].copy(), EYE_P, (6, 6))
    assert tuple(img2[2, 4]) == tuple(rgb[4])


def test_points_behind_the_camera_non_finite_or_off_screen_are_not_drawn():
    pts = _points([[2, 2, -1.0], [2, 2, 0.0], [3, 3, 1.0], [100, 2, 1.0], [2, -9, 1.0]])
    pts = np.concatenate([pts, [[np.nan, 2, 1], [2, np.inf, 1], [2, 2, np.nan]]]).astype(np.float32)
    _, depth, _ = O.render_points(pts, np.full((len(pts), 3), 9, np.uint8), EYE_P, (6, 6))
    assert _drawn(depth) == [(3, 3)]


@pytest.mark.parametrize("size, u, want", [(2, 2.0, [1, 2]), (2, 2.5, [2, 3]), (3, 2.0, [1, 2, 3]),
                                           (3, 2.5, [1, 2, 3]), (3, 2.6, [2, 3, 4]), (3, 0.2, [0, 1])])
def test_point_sizes_cover_the_expected_pixels(size, u, want):
    _, depth, _ = O.render_points(_points([[u, u, 1.0]]), [[1, 2, 3]], EYE_P, (8, 8), size)
    assert _drawn(depth) == sorted((x, y) for y in want for x in want)


# ---------------------------------------------------------------------------- restatement: triangles
def _tri(uv, w):
    return _points([[u, v, w] for u, v in uv])


@pytest.mark.parametrize("order", [(0, 1, 2), (0, 2, 1)])      # both windings
def test_screen_aligned_triangle_covers_its_edge_function_pixels(order):
    uv = [(1.0, 1.0), (5.0, 1.0), (1.0, 5.0)]
    verts = _tri(uv, 2.0)
    faces = np.array([order], np.int32)
    img, depth, _ = O.render_mesh(verts, np.full((3, 3), 200, np.uint8), faces, EYE_P,
                                  np.zeros(3, np.float32), (8, 7))
    want = [(x, y) for y in range(7) for x in range(8) if x >= 1 and y >= 1 and x + y <= 6]
    assert _drawn(depth) == sorted(want)
    assert (depth[depth > 0] == 2.0).all()                   # fronto-parallel: constant depth
    # the normal is the viewing axis, the centroid off it: shade = 0.3 + 0.7 cos
    g = verts.mean(0)
    cos = g[2] / np.linalg.norm(g)
    assert (np.abs(img[depth > 0].astype(int) - round(200 * (0.3 + 0.7 * cos))) <= 1).all()


def test_fronto_parallel_depth_is_constant_to_rounding():
    rng = np.random.default_rng(1)
    for _ in range(20):
        uv = rng.uniform(0, 40, (3, 2))
        w = rng.uniform(0.5, 50)
        _, depth, _ = O.render_mesh(_tri(uv, w), np.zeros((3, 3), np.uint8), [[0, 1, 2]], EYE_P,
                                    np.zeros(3, np.float32), (40, 40))
        d = depth[depth > 0].astype(np.float64)
        if len(d):
            assert np.abs(d - np.float32(w)).max() <= 4 * np.spacing(np.float32(w)), w


def test_triangles_nearer_win_and_skips():
    verts = np.concatenate([_tri([(0, 0), (9, 0), (0, 9)], 2.0), _tri([(0, 0), (9, 0), (0, 9)], 1.0),
                            _tri([(0, 0), (9, 0), (0, 9)], 1.0),
                            _tri([(1, 1), (2, 2), (3, 3)], 0.5),       # zero area
                            _tri([(0, 0), (9, 0), (0, 9)], 0.25)])
    verts[14, 2] = -1.0                                                # a vertex behind the camera
    faces = np.arange(15, dtype=np.int32).reshape(5, 3)
    col = np.repeat(np.array([[10], [20], [30], [40], [50]], np.uint8), 9, 0).reshape(15, 3)
    _, depth, zbuf = O.render_mesh(verts, col, faces, EYE_P, np.zeros(3, np.float32), (10, 10))
    won = (zbuf[zbuf != O.EMPTY] & np.uint64(0xFFFFFFFF)).astype(int)
    assert set(won) == {1}                                   # nearer than 0, ties 2, others skipped
    assert (depth[depth > 0] == 1.0).all()
    with pytest.raises(ValueError, match="outside"):
        O.render_mesh(verts, col, [[0, 1, 15]], EYE_P, np.zeros(3, np.float32), (10, 10))


# ---------------------------------------------------------------------------- entry points
def test_entry_points_refuse_bad_arguments_before_device_work():
    import ctypes

    from casmvsnet_pl_b200 import _lib
    lib = _lib.load()
    ok, odd4, odd2 = ctypes.c_void_p(0x10000), ctypes.c_void_p(0x10004), ctypes.c_void_p(0x10002)
    P = np.eye(4, dtype=np.float32)
    Pp = P.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    eye = np.zeros(3, np.float32).ctypes.data_as(ctypes.POINTER(ctypes.c_float))

    def refused(rc, what):
        msg = lib.casmvs_last_error()
        assert rc < 0 and what in msg, (rc, msg)

    def pts(xyz=ok, n=10, W=64, H=48, s=1, zbuf=ok, depth=ok):
        return lib.casmvs_render_points_fwd(xyz, ok, n, Pp, W, H, s, zbuf, ok, depth, None)
    refused(pts(xyz=odd2), b"xyz must be 4-byte aligned")
    refused(pts(zbuf=odd4), b"zbuf must be 8-byte aligned")
    refused(pts(depth=odd2), b"depth must be 4-byte aligned")
    refused(pts(n=1 << 32), b"n < 2^32")
    refused(pts(n=-1), b"n < 2^32")
    for W, H in ((0, 48), (64, 16385), (16385, 1)):
        refused(pts(W=W, H=H), b"1..16384")
    for s in (0, 65):
        refused(pts(s=s), b"point_size must lie in 1..64")
    refused(pts(xyz=None), b"null")
    ws = lib.casmvs_render_mesh_workspace_bytes(100)
    assert ws >= 100 * 4

    def tris(verts=ok, faces=ok, W=64, H=48, ws_bytes=ws, zbuf=ok, work=ok):
        return lib.casmvs_render_mesh_fwd(verts, ok, 10, faces, 100, Pp, eye, W, H, zbuf, work,
                                          ws_bytes, ok, ok, None)
    refused(tris(verts=odd2), b"verts must be 4-byte aligned")
    refused(tris(faces=odd2), b"faces must be 4-byte aligned")
    refused(tris(zbuf=odd4), b"zbuf must be 8-byte aligned")
    refused(tris(W=16385), b"1..16384")
    refused(tris(ws_bytes=ws - 1), b"workspace")
    refused(tris(work=None), b"null")


# ---------------------------------------------------------------------------- command line
def _oracle_draw(xyz, rgb, faces, P, wh, point_size=1):
    if faces is None:
        img, depth, _ = O.render_points(xyz, rgb, P, wh, point_size)
    else:
        img, depth, _ = O.render_mesh(xyz, rgb, faces, P, render.camera_centre(P), wh)
    return img, depth


@pytest.fixture
def oracle_renderer(monkeypatch):
    monkeypatch.setattr(render, "draw", _oracle_draw)


def _cloud(n=4000, seed=0):
    rng = np.random.default_rng(seed)
    xyz = rng.normal(size=(n, 3)).astype(np.float32) * [1, 0.5, 0.3]
    return xyz.astype(np.float32), rng.integers(0, 256, (n, 3), dtype=np.uint8)


def test_cli_arguments():
    a = render.parse_args(["--dataset_name", "tanks", "--scan", "Horse"])
    assert a.out_dir == os.path.join("results", "tanks") and a.point_size == 1
    assert not (a.mesh or a.use_viewpoint or a.save_viewpoint)
    for bad in (["--scan", "x"], ["--dataset_name", "dtu"], ["--dataset_name", "eth3d", "--scan", "x"],
                ["--dataset_name", "dtu", "--scan", "x", "--point_size", "0"],
                ["--dataset_name", "dtu", "--scan", "x", "--point_size", "65"]):
        with pytest.raises(SystemExit):
            render.parse_args(bad)


def test_cli_missing_files_name_the_path(tmp_path, oracle_renderer):
    base = ["--dataset_name", "dtu", "--scan", "scan9", "--out", str(tmp_path)]
    with pytest.raises(SystemExit, match=os.path.join("points", "scan9.ply")):
        render.main(base)
    with pytest.raises(SystemExit, match=os.path.join("mesh", "scan9.ply")):
        render.main(base + ["--mesh"])
    os.makedirs(tmp_path / "points")
    fusion.write_ply(str(tmp_path / "points" / "scan9.ply"), *_cloud(100))
    with pytest.raises(SystemExit, match="viewpoint.json"):
        render.main(base + ["--use_viewpoint"])
    (tmp_path / "viewpoint.json").write_text('{"class_name": "PinholeCameraParameters"}')
    with pytest.raises(SystemExit, match="'version_major'"):
        render.main(base + ["--use_viewpoint"])


def test_cli_viewpoints_and_outputs(tmp_path, oracle_renderer, capsys):
    from PIL import Image
    out = tmp_path / "res"
    os.makedirs(out / "points")
    xyz, rgb = _cloud()
    fusion.write_ply(str(out / "points" / "s1.ply"), xyz, rgb)
    base = ["--dataset_name", "colmap", "--scan", "s1", "--out", str(out)]
    png = render.main(base + ["--save_viewpoint"])
    assert png == os.path.join(str(out), "render", "s1.png")
    K, E = render.default_view(xyz)
    assert render.read_camera(str(out / "viewpoint.json"))[2] == (1920, 1080)
    want, _ = _oracle_draw(xyz, rgb, None, render.projection(K, E), (1920, 1080))
    assert np.array_equal(np.asarray(Image.open(png)), want)
    assert "s1 contains 0.00 M points" in capsys.readouterr().out
    # an edited viewpoint is used at its own size, also when --save_viewpoint is given too
    K2 = np.array([[300.0, 0, 199.5], [0, 300.0, 149.5], [0, 0, 1]])
    render.write_viewpoint(str(out / "viewpoint.json"), K2, E, (400, 300))
    before = (out / "viewpoint.json").read_bytes()
    png = render.main(base + ["--use_viewpoint", "--save_viewpoint", "--point_size", "3"])
    assert (out / "viewpoint.json").read_bytes() == before
    want, depth = _oracle_draw(xyz, rgb, None, render.projection(K2, E), (400, 300), 3)
    assert np.array_equal(np.asarray(Image.open(png)), want)
    assert f"{int((depth > 0).sum())} of 120000 pixels drawn" in capsys.readouterr().out


def test_cli_cloud_without_colours_renders_white(tmp_path, oracle_renderer):
    out = tmp_path / "r"
    os.makedirs(out / "points")
    xyz, _ = _cloud(500)
    header = (f"ply\nformat ascii 1.0\nelement vertex {len(xyz)}\nproperty float x\n"
              "property float y\nproperty float z\nend_header\n")
    rows = "\n".join(" ".join(repr(float(c)) for c in p) for p in xyz)
    (out / "points" / "w.ply").write_text(header + rows + "\n")
    from PIL import Image
    img = np.asarray(Image.open(render.main(["--dataset_name", "dtu", "--scan", "w", "--out", str(out)])))
    drawn = (img != O.BACKGROUND).any(-1)
    assert drawn.sum() > 100 and (img[drawn] == 255).all()


def test_cli_mesh(tmp_path, oracle_renderer, capsys):
    from PIL import Image
    out = tmp_path / "m"
    os.makedirs(out / "mesh")
    # an octahedron, coloured per vertex
    v = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)
    f = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5],
                  [0, 3, 5]], np.int32)
    c = (np.abs(v) * 200 + 20).astype(np.uint8)
    mesh.write_mesh_ply(str(out / "mesh" / "oct.ply"), v, c, f)
    png = render.main(["--dataset_name", "tanks", "--scan", "oct", "--mesh", "--out", str(out)])
    assert png.endswith(os.path.join("render", "oct_mesh.png"))
    K, E = render.default_view(v)
    want, depth = _oracle_draw(v, c, f, render.projection(K, E), (1920, 1080))
    assert np.array_equal(np.asarray(Image.open(png)), want)
    assert (depth > 0).sum() > 100_000
    assert "oct contains 8 triangles" in capsys.readouterr().out
