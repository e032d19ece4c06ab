"""Render fused point clouds and meshes to images on the GPU, without a display (csrc/render.cu;
float32 numpy restatement in oracle/render_oracle.py, bit for bit).

    image, depth = render_points(xyz, rgb, P, (W, H), point_size=1)
    image, depth = render_mesh(verts, colours, faces, P, (W, H))
    image, depth = render_textured_mesh(verts, faces, uv, page, atlas, P, (W, H))

take CUDA tensors ((N,3) float32 positions, (N,3) uint8 colours, (M,3) int32 faces) and a 4x4
world -> pixel matrix P, and return (H,W,3) uint8 and (H,W) float32 camera depth (0 where nothing
is drawn) on the device.  The nearest primitive wins a pixel and an exact depth tie goes to the
lower index, so the same inputs give the same image on every run.  The background is
(128, 128, 255).  Points cover s x s pixels; triangles are drawn from both sides, shaded flat by
0.3 + 0.7 |cos| of the angle between their normal and the line of sight to their centroid, and
skipped whole when a vertex lies behind the camera (no near-plane clipping).

Viewpoints are Open3D PinholeCameraParameters JSON files, the format of the `viewpoint.json`
the original project's visualize_ply.py saves (read_viewpoint / write_viewpoint).  The command
line renders a scan the pipeline wrote:

    python -m casmvsnet_pl_b200.render --dataset_name dtu --scan scan9 \\
        [--use_viewpoint | --save_viewpoint] [--mesh [--textured]] [--point_size 1] [--out results/dtu]

A textured mesh (texture.py) is drawn unshaded: its UV is interpolated perspective-correctly and
its atlas page sampled bilinearly, texel centres at i + 0.5, indices clamped to the page.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import math
import os

import numpy as np
import torch

from . import _lib

BACKGROUND = (128, 128, 255)
DEFAULT_WH = (1920, 1080)
MAX_SIDE = 16384
MAX_POINT_SIZE = 64
FOV_Y = 60.0                      # degrees, the default view's vertical field of view
ZOOM = 0.7                        # default view: distance = ZOOM * max extent / tan(FOV_Y / 2)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check_cuda(name, t, dtype, cols):
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype == dtype and t.dim() == 2
            and t.shape[1] == cols):
        raise ValueError(f"{name} must be a {dtype} CUDA tensor of shape (N, {cols})")
    return t.contiguous()


def _matrix(P):
    P = np.asarray(P, dtype=np.float32)
    if P.shape != (4, 4) or not np.isfinite(P).all():
        raise ValueError("P must be a finite 4x4 world -> pixel matrix")
    return np.ascontiguousarray(P)


def _size(wh):
    W, H = (int(x) for x in wh)
    if not (1 <= W <= MAX_SIDE and 1 <= H <= MAX_SIDE):
        raise ValueError(f"image size must lie in 1..{MAX_SIDE} per side, got {W}x{H}")
    return W, H


def _f32p(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def camera_centre(P):
    """The camera centre of a world -> pixel matrix (float32 P, solved in float64) as float32:
    the eye of the mesh shade."""
    P = _matrix(P).astype(np.float64)
    return (-np.linalg.solve(P[:3, :3], P[:3, 3])).astype(np.float32)


def _outputs(W, H, device):
    return (torch.empty(H * W, dtype=torch.int64, device=device),
            torch.empty(H, W, 3, dtype=torch.uint8, device=device),
            torch.empty(H, W, dtype=torch.float32, device=device))


def render_points(xyz, rgb, P, wh, point_size=1):
    """Points (N,3) float32 with colours (N,3) uint8, CUDA tensors -> (image (H,W,3) uint8,
    depth (H,W) float32) on their device.  A point of size s (1..64) covers the pixels whose
    integer centres lie in [u - s/2, u + s/2) x [v - s/2, v + s/2)."""
    xyz = _check_cuda("xyz", xyz, torch.float32, 3)
    rgb = _check_cuda("rgb", rgb, torch.uint8, 3)
    if len(rgb) != len(xyz) or rgb.device != xyz.device:
        raise ValueError("rgb must hold one colour per point, on the points' device")
    if not (isinstance(point_size, int) and 1 <= point_size <= MAX_POINT_SIZE):
        raise ValueError(f"point_size must be an integer in 1..{MAX_POINT_SIZE}, got {point_size}")
    W, H = _size(wh)
    P = _matrix(P)
    with torch.cuda.device(xyz.device):
        zbuf, image, depth = _outputs(W, H, xyz.device)
        _lib.check(_lib.load().casmvs_render_points_fwd(
            _ptr(xyz), _ptr(rgb), len(xyz), _f32p(P), W, H, point_size, _ptr(zbuf), _ptr(image),
            _ptr(depth), _stream()), "render_points_fwd")
    return image, depth


def render_mesh(verts, colours, faces, P, wh):
    """Triangles faces (M,3) int32 over verts (N,3) float32 with colours (N,3) uint8, CUDA
    tensors -> (image (H,W,3) uint8, depth (H,W) float32) on their device.  Colours are
    interpolated perspective-correctly and shaded flat and two-sided; a face index outside
    [0, N) raises CasMVSError."""
    verts = _check_cuda("verts", verts, torch.float32, 3)
    colours = _check_cuda("colours", colours, torch.uint8, 3)
    faces = _check_cuda("faces", faces, torch.int32, 3)
    if len(colours) != len(verts) or not (colours.device == faces.device == verts.device):
        raise ValueError("colours must hold one colour per vertex, on one device with the faces")
    W, H = _size(wh)
    P = _matrix(P)
    eye = camera_centre(P)
    lib = _lib.load()
    with torch.cuda.device(verts.device):
        zbuf, image, depth = _outputs(W, H, verts.device)
        nbytes = lib.casmvs_render_mesh_workspace_bytes(len(faces))
        ws = torch.empty((nbytes + 3) // 4, dtype=torch.int32, device=verts.device)
        _lib.check(lib.casmvs_render_mesh_fwd(
            _ptr(verts), _ptr(colours), len(verts), _ptr(faces), len(faces), _f32p(P), _f32p(eye),
            W, H, _ptr(zbuf), _ptr(ws), ws.numel() * 4, _ptr(image), _ptr(depth), _stream()),
            "render_mesh_fwd")
    return image, depth


def render_textured_mesh(verts, faces, uv, page, atlas, P, wh):
    """Triangles faces (M,3) int32 over verts (N,3) float32 with per-corner uv (M,3,2) float32,
    a page (M,) int32 per face and atlas (pages,S,S,3) uint8, CUDA tensors (texture.texture_mesh
    returns them) -> (image (H,W,3) uint8, depth (H,W) float32) on their device.  The raster
    pass is render_mesh's; the colour is the page sampled bilinearly at the perspective-correct UV,
    unshaded (the photographs carry the light)."""
    verts = _check_cuda("verts", verts, torch.float32, 3)
    faces = _check_cuda("faces", faces, torch.int32, 3)
    if not (torch.is_tensor(uv) and uv.is_cuda and uv.dtype == torch.float32
            and tuple(uv.shape) == (len(faces), 3, 2)):
        raise ValueError("uv must be a float32 CUDA tensor of shape (M, 3, 2)")
    if not (torch.is_tensor(page) and page.is_cuda and page.dtype == torch.int32
            and tuple(page.shape) == (len(faces),)):
        raise ValueError("page must be an int32 CUDA tensor of shape (M,)")
    if not (torch.is_tensor(atlas) and atlas.is_cuda and atlas.dtype == torch.uint8
            and atlas.dim() == 4 and atlas.shape[1] == atlas.shape[2] and atlas.shape[3] == 3
            and len(atlas) >= 1 and atlas.shape[1] <= MAX_SIDE):
        raise ValueError(f"atlas must be a uint8 CUDA tensor of shape (pages, S, S, 3), S <= {MAX_SIDE}")
    if not (verts.device == faces.device == uv.device == page.device == atlas.device):
        raise ValueError("the mesh, its UVs, pages and atlas must be on one device")
    if len(page) and not bool(((page >= 0) & (page < len(atlas))).all()):
        raise ValueError(f"page holds an index outside 0..{len(atlas) - 1}")
    W, H = _size(wh)
    P = _matrix(P)
    uv, page, atlas = uv.contiguous(), page.contiguous(), atlas.contiguous()
    lib = _lib.load()
    with torch.cuda.device(verts.device):
        zbuf, image, depth = _outputs(W, H, verts.device)
        nbytes = lib.casmvs_render_mesh_workspace_bytes(len(faces))
        ws = torch.empty((nbytes + 3) // 4, dtype=torch.int32, device=verts.device)
        _lib.check(lib.casmvs_render_textured_mesh_fwd(
            _ptr(verts), len(verts), _ptr(faces), len(faces), _ptr(uv), _ptr(page), _ptr(atlas),
            len(atlas), atlas.shape[1], _f32p(P), W, H, _ptr(zbuf), _ptr(ws), ws.numel() * 4,
            _ptr(image), _ptr(depth), _stream()), "render_textured_mesh_fwd")
    return image, depth


def draw(xyz, rgb, faces, P, wh, point_size=1, device="cuda"):
    """Host arrays in, host arrays out: uploads, renders the points (faces None) or the mesh,
    and downloads (image (H,W,3) uint8, depth (H,W) float32)."""
    x = torch.from_numpy(np.ascontiguousarray(xyz, np.float32)).to(device)
    c = torch.from_numpy(np.ascontiguousarray(rgb, np.uint8)).to(device)
    if faces is None:
        image, depth = render_points(x, c, P, wh, point_size)
    else:
        f = torch.from_numpy(np.ascontiguousarray(faces, np.int32)).to(device)
        image, depth = render_mesh(x, c, f, P, wh)
    return image.cpu().numpy(), depth.cpu().numpy()


# ---------------------------------------------------------------------------- viewpoints
def projection(K, E):
    """4x4 world -> pixel matrix [K 0; 0 1] @ E (float64)."""
    K4 = np.eye(4)
    K4[:3, :3] = np.asarray(K, dtype=np.float64)
    return K4 @ np.asarray(E, dtype=np.float64)


def _numbers(path, data, key, n):
    v = data.get(key.rsplit(".", 1)[-1]) if isinstance(data, dict) else None
    if not (isinstance(v, list) and len(v) == n
            and all(isinstance(x, (int, float)) and not isinstance(x, bool) for x in v)
            and all(math.isfinite(x) for x in v)):
        raise ValueError(f"{path}: '{key}' must be a list of {n} finite numbers")
    return np.array(v, dtype=np.float64)


def read_camera(path):
    """An Open3D PinholeCameraParameters JSON file -> (K (3,3), E (4,4) world -> camera, both
    float64, (W, H)).  `extrinsic` (16 numbers) and `intrinsic.intrinsic_matrix` (9 numbers) are
    column-major.  Any pinhole K (last row 0 0 1, fx, fy > 0) is read.  A file that does not
    match the schema raises ValueError naming the key."""
    try:
        with open(path) as f:
            data = json.load(f)
    except json.JSONDecodeError as e:
        raise ValueError(f"{path}: not a JSON file ({e})") from None
    if not isinstance(data, dict):
        raise ValueError(f"{path}: a viewpoint file holds one JSON object")
    if data.get("class_name") != "PinholeCameraParameters":
        raise ValueError(f"{path}: 'class_name' must be 'PinholeCameraParameters'")
    for key, want in (("version_major", 1), ("version_minor", 0)):
        if data.get(key) != want or isinstance(data.get(key), bool):
            raise ValueError(f"{path}: '{key}' must be {want}")
    E = _numbers(path, data, "extrinsic", 16).reshape(4, 4, order="F")
    if not np.array_equal(E[3], [0, 0, 0, 1]):
        raise ValueError(f"{path}: 'extrinsic' must end in the row 0 0 0 1")
    intr = data.get("intrinsic")
    if not isinstance(intr, dict):
        raise ValueError(f"{path}: 'intrinsic' must be an object")
    wh = []
    for key in ("width", "height"):
        v = intr.get(key)
        if not (isinstance(v, int) and not isinstance(v, bool) and v >= 1):
            raise ValueError(f"{path}: 'intrinsic.{key}' must be a positive integer")
        wh.append(v)
    K = _numbers(path, intr, "intrinsic.intrinsic_matrix", 9).reshape(3, 3, order="F")
    if not (np.array_equal(K[2], [0, 0, 1]) and K[0, 0] > 0 and K[1, 1] > 0):
        raise ValueError(f"{path}: 'intrinsic.intrinsic_matrix' must be a pinhole matrix "
                         "(last row 0 0 1, fx > 0, fy > 0)")
    return K, E, tuple(wh)


def read_viewpoint(path):
    """-> (P (4,4) float64 world -> pixel, (W, H)) of a viewpoint file (see read_camera)."""
    K, E, wh = read_camera(path)
    return projection(K, E), wh


def write_viewpoint(path, K, E, wh):
    """Write K, E and the image size as Open3D PinholeCameraParameters JSON.  Only what Open3D
    reads back is written: fx == fy, no skew, cx = W/2 - 0.5, cy = H/2 - 0.5; anything else
    raises ValueError."""
    K = np.asarray(K, dtype=np.float64)
    E = np.asarray(E, dtype=np.float64)
    W, H = (int(x) for x in wh)
    if K.shape != (3, 3) or E.shape != (4, 4) or not (np.isfinite(K).all() and np.isfinite(E).all()):
        raise ValueError("K must be a finite 3x3 and E a finite 4x4 matrix")
    if not (W >= 1 and H >= 1):
        raise ValueError(f"image size must be positive, got {W}x{H}")
    if not (K[0, 0] == K[1, 1] > 0 and K[0, 1] == K[1, 0] == 0 and np.array_equal(K[2], [0, 0, 1])
            and K[0, 2] == W / 2 - 0.5 and K[1, 2] == H / 2 - 0.5):
        raise ValueError("Open3D reads back only fx == fy, zero skew and the principal point "
                         f"(W/2 - 0.5, H/2 - 0.5) = ({W / 2 - 0.5}, {H / 2 - 0.5})")
    if not np.array_equal(E[3], [0, 0, 0, 1]):
        raise ValueError("E must end in the row 0 0 0 1")
    data = {"class_name": "PinholeCameraParameters",
            "extrinsic": [float(x) for x in E.reshape(-1, order="F")],
            "intrinsic": {"height": H, "intrinsic_matrix": [float(x) for x in K.reshape(-1, order="F")],
                          "width": W},
            "version_major": 1, "version_minor": 0}
    with open(path, "w") as f:
        json.dump(data, f, indent=4)
        f.write("\n")


def default_view(xyz, wh=DEFAULT_WH):
    """The initial view of Open3D's visualiser, as this project's rule -> (K, E) float64.
    It looks at the centre of the finite points' axis-aligned bounding box along -z
    (front (0, 0, 1), up (0, 1, 0)) from ZOOM * max extent / tan(FOV_Y / 2) away (a max extent
    of 0 counts as 1), with fx = fy = (H/2) / tan(FOV_Y / 2) and the principal point
    (W/2 - 0.5, H/2 - 0.5).  Camera axes: x = right, y = -up, z = -front."""
    W, H = _size(wh)
    if torch.is_tensor(xyz):
        x = xyz.reshape(-1, 3)
        x = x[torch.isfinite(x).all(1)]
        lo, hi = ((x.amin(0), x.amax(0)) if len(x) else (torch.zeros(3),) * 2)
        lo, hi = lo.double().cpu().numpy(), hi.double().cpu().numpy()
    else:
        x = np.asarray(xyz).reshape(-1, 3)
        x = x[np.isfinite(x).all(1)]
        lo, hi = (x.min(0), x.max(0)) if len(x) else (np.zeros(3),) * 2
        lo, hi = lo.astype(np.float64), hi.astype(np.float64)
    lookat = (lo + hi) / 2
    extent = float((hi - lo).max())
    t = math.tan(math.radians(FOV_Y / 2))
    dist = ZOOM * (extent if extent > 0 else 1.0) / t
    front, up = np.array([0.0, 0.0, 1.0]), np.array([0.0, 1.0, 0.0])
    right = np.cross(up, front)
    R = np.stack([right, -up, -front])
    eye = lookat + dist * front
    E = np.eye(4)
    E[:3, :3], E[:3, 3] = R, -R @ eye
    f = (H / 2) / t
    K = np.array([[f, 0, W / 2 - 0.5], [0, f, H / 2 - 0.5], [0, 0, 1.0]])
    return K, E


# ---------------------------------------------------------------------------- command line
def parse_args(argv=None):
    ap = argparse.ArgumentParser(
        description="Render <out>/points/<scan>.ply (or <out>/mesh/<scan>.ply with --mesh) to "
                    "<out>/render/<scan>.png (<scan>_mesh.png) on the GPU.")
    ap.add_argument("--dataset_name", required=True, choices=["dtu", "tanks", "blendedmvs", "colmap"])
    ap.add_argument("--scan", required=True)
    ap.add_argument("--use_viewpoint", action="store_true",
                    help="render from <out>/viewpoint.json at that file's image size")
    ap.add_argument("--save_viewpoint", action="store_true",
                    help="write the default view to <out>/viewpoint.json (ignored with --use_viewpoint)")
    ap.add_argument("--mesh", action="store_true", help="render the mesh of eval_pipeline --mesh")
    ap.add_argument("--textured", action="store_true",
                    help="with --mesh: draw the textured <out>/mesh/<scan>.obj of eval_pipeline "
                         "--mesh_texture to <out>/render/<scan>_textured.png")
    ap.add_argument("--point_size", type=int, default=1, help=f"pixels per side, 1..{MAX_POINT_SIZE}")
    ap.add_argument("--out", default=None, help="output directory (default results/<dataset_name>)")
    a = ap.parse_args(argv)
    if a.textured and not a.mesh:
        ap.error("--textured needs --mesh")
    if not 1 <= a.point_size <= MAX_POINT_SIZE:
        ap.error(f"--point_size must lie in 1..{MAX_POINT_SIZE}")
    a.out_dir = a.out or os.path.join("results", a.dataset_name)
    return a


def load_scan(path, mesh):
    """-> (xyz (N,3) float32, rgb (N,3) uint8, faces (M,3) int32 or None) of a point or mesh
    PLY; a cloud without red / green / blue is white."""
    from . import io as cio
    if mesh:
        return cio.read_mesh_ply(path)
    v = cio.read_ply(path)
    names = v.dtype.names
    if not {"x", "y", "z"} <= set(names):
        raise ValueError(f"{path}: the vertices have no x, y, z")
    xyz = np.stack([v["x"], v["y"], v["z"]], 1).astype(np.float32)
    if {"red", "green", "blue"} <= set(names):
        rgb = np.stack([v["red"], v["green"], v["blue"]], 1).astype(np.uint8)
    else:
        rgb = np.full((len(v), 3), 255, np.uint8)
    return xyz, rgb, None


def main(argv=None):
    """-> the path of the PNG written."""
    a = parse_args(argv)
    kind = "mesh" if a.mesh else "points"
    ply = os.path.join(a.out_dir, kind, f"{a.scan}.obj" if a.textured else f"{a.scan}.ply")
    vp = os.path.join(a.out_dir, "viewpoint.json")
    if not os.path.isfile(ply):
        raise SystemExit(f"{ply}: no such file")
    if a.use_viewpoint and not os.path.isfile(vp):
        raise SystemExit(f"{vp}: no such file (write one with --save_viewpoint)")
    if a.textured:
        from . import texture
        xyz, faces, uv, page, atlas = texture.read_textured_obj(ply)
        rgb = None
    else:
        xyz, rgb, faces = load_scan(ply, a.mesh)
    if a.use_viewpoint:
        try:
            P, wh = read_viewpoint(vp)
        except ValueError as e:
            raise SystemExit(str(e)) from None
    else:
        wh = DEFAULT_WH
        K, E = default_view(xyz, wh)
        P = projection(K, E)
        if a.save_viewpoint:
            write_viewpoint(vp, K, E, wh)
            print(f"viewpoint saved to {vp}")
    if a.textured:
        def cuda(x):
            return torch.from_numpy(np.ascontiguousarray(x)).to("cuda")
        image, depth = render_textured_mesh(cuda(xyz), cuda(faces), cuda(uv), cuda(page),
                                            cuda(atlas), P, wh)
        image, depth = image.cpu().numpy(), depth.cpu().numpy()
    else:
        image, depth = draw(xyz, rgb, faces, P, wh, a.point_size)
    from PIL import Image
    os.makedirs(os.path.join(a.out_dir, "render"), exist_ok=True)
    png = os.path.join(a.out_dir, "render", f"{a.scan}_textured.png" if a.textured else
                       f"{a.scan}_mesh.png" if a.mesh else f"{a.scan}.png")
    Image.fromarray(image).save(png)
    what = (f"{len(faces)} triangles" if a.mesh else f"{len(xyz) / 1e6:.2f} M points")
    print(f"{a.scan} contains {what}; {int((depth > 0).sum())} of {wh[0] * wh[1]} pixels drawn "
          f"-> {png}")
    return png


if __name__ == "__main__":
    main()
