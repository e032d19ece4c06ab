"""Scenes reconstructed with COLMAP, as the input of eval_pipeline --dataset_name colmap.

The input is the workspace `colmap image_undistorter` writes, or a `colmap mapper` project:

    <root>/images/<name>                          the images (or any directory: --image_dir)
    <root>/sparse/{cameras,images,points3D}.bin   (or .txt; or under <root>/sparse/0) the model

Conversion, in order:

  read_model         the model in COLMAP's binary or text format (host).  By default only the
                     undistorted camera models PINHOLE and SIMPLE_PINHOLE are accepted;
                     distorted=True also admits the seven DISTORTED_MODELS.  Everything the files
                     supply is validated before anything reaches the GPU: finite poses, intrinsics
                     and points, tracks that name registered images, and for a distorted camera
                     its undistorted camera (undistorted_camera).
  undistorted_camera the PINHOLE camera a distorted one is resampled to (README, "Your own
                     scene"): the border pixels undistorted by Newton's method in float64, the
                     scales of the largest centred box they enclose clipped to [0.2, 2], the size
                     and principal point scaled by them.  The images are undistorted on the GPU
                     as they are read (io.undistort_u8, csrc/undistort.cu).
  load_scene         views 0..n-1 in sorted image-name order: full-resolution K, world->camera
                     E = [R(q) | t], camera centre c = -R^T t, tracks in CSR form over view ids
                     (an image listed twice in one track counts once).
  view_scores        the MVSNet paper's view-selection score of every image pair
                     (casmvs_view_scores_fwd, csrc/view_select.cu, double, deterministic).
  depth_stats        z of every observed point in its own camera, per-view sort and percentile
                     picks: torch ops on the device.
  select_sources / assemble
                     each view's sources (the n_src best views with a positive score, by score
                     descending, lower id first on a tie), the reference views kept, and each
                     one's depth range:
                         depth_min = 0.75 * q(0.01),  depth_max = 1.25 * q(0.99)
                     over the view's observed points with z > 0, where q(f) is the element at
                     index floor(f * (n - 1)) of their ascending sort.  Sparse points under-sample
                     a surface's extremes, so the range is widened by this project's rule.
  write_cams / write_pair / write_view_names
                     the record of a run: MVSNet cam files, pair.txt with the scores, and the
                     view id -> image name map.
"""
from __future__ import annotations

import os
import struct

import numpy as np
import torch

# COLMAP's camera models: id -> (name, number of parameters)
CAMERA_MODELS = {0: ("SIMPLE_PINHOLE", 3), 1: ("PINHOLE", 4), 2: ("SIMPLE_RADIAL", 4),
                 3: ("RADIAL", 5), 4: ("OPENCV", 8), 5: ("OPENCV_FISHEYE", 8),
                 6: ("FULL_OPENCV", 12), 7: ("FOV", 5), 8: ("SIMPLE_RADIAL_FISHEYE", 4),
                 9: ("RADIAL_FISHEYE", 5), 10: ("THIN_PRISM_FISHEYE", 12)}
MODEL_IDS = {name: (i, n) for i, (name, n) in CAMERA_MODELS.items()}
SUPPORTED_MODELS = ("PINHOLE", "SIMPLE_PINHOLE")
DISTORTED_MODELS = ("SIMPLE_RADIAL", "RADIAL", "OPENCV", "FULL_OPENCV", "SIMPLE_RADIAL_FISHEYE",
                    "RADIAL_FISHEYE", "OPENCV_FISHEYE")
FISHEYE_MODELS = ("SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE", "OPENCV_FISHEYE")
SINGLE_FOCAL_MODELS = ("SIMPLE_PINHOLE", "SIMPLE_RADIAL", "RADIAL", "SIMPLE_RADIAL_FISHEYE",
                       "RADIAL_FISHEYE")
UNDISTORT_SCALES = (0.2, 2.0)       # min_scale, max_scale of the undistorted camera
NEWTON_ITERS = 100
NEWTON_TOL_PX = 1e-9                # round-trip residual a border pixel must reach

N_SRC = 10                 # sources listed per view
MIN_FRONT_POINTS = 20      # a reference view needs this many observed points in front of it
DEPTH_QUANTILES = (0.01, 0.99)
DEPTH_WIDEN = (0.75, 1.25)


class ColmapModel:
    """A COLMAP model as read: cameras {camera_id: (model, width, height, params)}, images
    {image_id: (qvec (4,) wxyz, tvec (3,), camera_id, name)}, point ids (N,) int64, xyz (N,3)
    float64 and the tracks as COLMAP image ids in CSR form: point k is seen by
    track_img[track_ptr[k]:track_ptr[k+1]] (int64)."""

    def __init__(self, cameras, images, point_ids, xyz, track_ptr, track_img):
        self.cameras, self.images = cameras, images
        self.point_ids = np.asarray(point_ids, np.int64)
        self.xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
        self.track_ptr = np.asarray(track_ptr, np.int64)
        self.track_img = np.asarray(track_img, np.int64)


# ------------------------------------------------------------------------------ reading
def _read_cameras_bin(path):
    cams = {}
    with open(path, "rb") as f:
        buf = f.read()
    (n,), off = struct.unpack_from("<Q", buf, 0), 8
    for _ in range(n):
        cid, mid, w, h = struct.unpack_from("<iiQQ", buf, off)
        off += 24
        if mid not in CAMERA_MODELS:
            raise ValueError(f"{path}: unknown camera model id {mid}")
        name, k = CAMERA_MODELS[mid]
        cams[cid] = (name, int(w), int(h), np.array(struct.unpack_from(f"<{k}d", buf, off)))
        off += 8 * k
    return cams


def _read_cameras_txt(path):
    cams = {}
    for line in _lines(path):
        tok = line.split()
        name = tok[1]
        if name not in MODEL_IDS:
            raise ValueError(f"{path}: unknown camera model {name}")
        params = np.array([float(x) for x in tok[4:]])
        if len(params) != MODEL_IDS[name][1]:
            raise ValueError(f"{path}: camera {tok[0]} ({name}) has {len(params)} parameters")
        cams[int(tok[0])] = (name, int(tok[2]), int(tok[3]), params)
    return cams


def _read_images_bin(path):
    imgs = {}
    with open(path, "rb") as f:
        buf = f.read()
    (n,), off = struct.unpack_from("<Q", buf, 0), 8
    for _ in range(n):
        iid = struct.unpack_from("<i", buf, off)[0]
        v = struct.unpack_from("<7d", buf, off + 4)
        cid = struct.unpack_from("<i", buf, off + 60)[0]
        off += 64
        end = buf.index(b"\0", off)
        name = buf[off:end].decode("utf-8")
        off = end + 1
        n2d = struct.unpack_from("<Q", buf, off)[0]
        off += 8 + 24 * n2d                      # (x, y, point3D_id) per 2D point: not needed
        imgs[iid] = (np.array(v[:4]), np.array(v[4:]), cid, name)
    return imgs


def _read_images_txt(path):
    imgs = {}
    lines = _lines(path, keep_empty=True)
    for k in range(0, len(lines) - 1, 2):       # the pose line, then the 2D points line
        tok = lines[k].split()
        if len(tok) < 10:
            raise ValueError(f"{path}: malformed image line {lines[k]!r}")
        v = [float(x) for x in tok[1:8]]
        imgs[int(tok[0])] = (np.array(v[:4]), np.array(v[4:]), int(tok[8]), " ".join(tok[9:]))
    return imgs


def _read_points_bin(path):
    with open(path, "rb") as f:
        buf = f.read()
    n = struct.unpack_from("<Q", buf, 0)[0]
    starts, lens = np.empty(n, np.int64), np.empty(n, np.int64)
    off = 8
    for k in range(n):                           # records are variable-length: find them first
        starts[k] = off
        lens[k] = struct.unpack_from("<Q", buf, off + 43)[0]
        off += 51 + 8 * lens[k]
    raw = np.frombuffer(buf, np.uint8)
    rec = raw[starts[:, None] + np.arange(32)].copy() if n else np.zeros((0, 32), np.uint8)
    ids = rec[:, :8].copy().view("<u8").ravel().astype(np.int64)
    xyz = rec[:, 8:32].copy().view("<f8").reshape(-1, 3)
    ptr = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=ptr[1:])
    tstart = np.repeat(starts + 51, lens) + 8 * (np.arange(ptr[-1]) - np.repeat(ptr[:-1], lens))
    img = raw[tstart[:, None] + np.arange(4)].copy().view("<i4").ravel().astype(np.int64) \
        if len(tstart) else np.zeros(0, np.int64)
    return ids, xyz, ptr, img


def _read_points_txt(path):
    ids, xyz, lens, img = [], [], [], []
    for line in _lines(path):
        tok = line.split()
        track = tok[8:]
        if len(track) % 2:
            raise ValueError(f"{path}: point {tok[0]} has an odd track")
        ids.append(int(tok[0]))
        xyz.append([float(x) for x in tok[1:4]])
        lens.append(len(track) // 2)
        img.extend(int(x) for x in track[0::2])
    ptr = np.zeros(len(ids) + 1, np.int64)
    np.cumsum(lens, out=ptr[1:])
    return np.array(ids, np.int64), np.array(xyz, np.float64).reshape(-1, 3), ptr, \
        np.array(img, np.int64)


def _lines(path, keep_empty=False):
    with open(path) as f:
        out = [line.rstrip("\r\n") for line in f if not line.startswith("#")]
    return out if keep_empty else [line for line in out if line.strip()]


def find_sparse_dir(root):
    """The model directory: <root>/sparse (an undistorted workspace), <root> itself, or
    <root>/sparse/0 (where `colmap mapper` writes its first model)."""
    for d in (os.path.join(root, "sparse"), root, os.path.join(root, "sparse", "0")):
        for ext in (".bin", ".txt"):
            if os.path.isfile(os.path.join(d, "cameras" + ext)):
                return d
    raise FileNotFoundError(f"no COLMAP model (cameras.bin / cameras.txt) under {root}/sparse")


def read_model(sparse_dir, ext=None, distorted=False):
    """cameras, images and points3D of a COLMAP model, binary (.bin, preferred when both exist)
    or text (.txt), validated (check_model; `distorted` admits the DISTORTED_MODELS)."""
    if ext is None:
        ext = ".bin" if os.path.isfile(os.path.join(sparse_dir, "cameras.bin")) else ".txt"
    p = lambda name: os.path.join(sparse_dir, name + ext)      # noqa: E731
    if ext == ".bin":
        model = ColmapModel(_read_cameras_bin(p("cameras")), _read_images_bin(p("images")),
                            *_read_points_bin(p("points3D")))
    else:
        model = ColmapModel(_read_cameras_txt(p("cameras")), _read_images_txt(p("images")),
                            *_read_points_txt(p("points3D")))
    check_model(model, distorted)
    return model


def check_model(model, distorted=False):
    """Raises ValueError unless every camera is PINHOLE or SIMPLE_PINHOLE with finite positive
    focal lengths and a positive size (or, with `distorted`, one of DISTORTED_MODELS that
    undistorted_camera accepts), every image has a finite pose with a nonzero quaternion and an
    existing camera, every point is finite and every track entry names a registered image."""
    for cid, (name, w, h, params) in model.cameras.items():
        if name not in SUPPORTED_MODELS:
            if not distorted:
                raise ValueError(f"camera {cid} uses the {name} model; only undistorted PINHOLE and "
                                 "SIMPLE_PINHOLE cameras are supported: run `colmap image_undistorter` "
                                 "on the reconstruction first")
            if name not in DISTORTED_MODELS:
                raise ValueError(f"camera {cid} uses the {name} model, which is not supported; the "
                                 "supported models are " + ", ".join(SUPPORTED_MODELS + DISTORTED_MODELS))
            undistorted_camera(cid, name, w, h, params)
            continue
        if w <= 0 or h <= 0 or not np.all(np.isfinite(params)) or np.any(params[:1] <= 0):
            raise ValueError(f"camera {cid}: bad size or parameters")
    for iid, (q, t, cid, name) in model.images.items():
        if not (np.all(np.isfinite(q)) and np.all(np.isfinite(t))) or not np.any(q):
            raise ValueError(f"image {iid} ({name}): pose is not finite")
        if cid not in model.cameras:
            raise ValueError(f"image {iid} ({name}) uses camera {cid}, which the model lacks")
    if not np.all(np.isfinite(model.xyz)):
        raise ValueError("points3D: coordinates are not finite")
    ptr = model.track_ptr
    if len(ptr) != len(model.xyz) + 1 or ptr[0] != 0 or np.any(np.diff(ptr) < 0) \
            or ptr[-1] != len(model.track_img):
        raise ValueError("points3D: malformed tracks")
    known = np.array(sorted(model.images), np.int64)
    pos = np.searchsorted(known, model.track_img)
    bad = (pos >= len(known)) | (known[np.minimum(pos, max(len(known) - 1, 0))] != model.track_img) \
        if len(known) else np.ones(len(model.track_img), bool)
    if np.any(bad):
        k = int(np.argmax(bad))
        p = int(np.searchsorted(ptr, k, side="right") - 1)
        raise ValueError(f"points3D: point {model.point_ids[p]} has a track entry for image "
                         f"{model.track_img[k]}, which the model lacks")


# ------------------------------------------------------------------------------ writing
def write_model(sparse_dir, model, fmt="bin"):
    """Write `model` in COLMAP's binary ("bin") or text ("txt") format.  Each image lists one 2D
    point per track entry naming it (coordinates 0), and each track entry refers to it (a
    track entry naming an image the model lacks is written as it is, with 2D point index 0)."""
    os.makedirs(sparse_dir, exist_ok=True)
    obs = {iid: [] for iid in model.images}          # image id -> [point3D id]
    track_idx = np.zeros(len(model.track_img), np.int64)
    for k in range(len(model.xyz)):
        for e in range(model.track_ptr[k], model.track_ptr[k + 1]):
            lst = obs.get(int(model.track_img[e]), [])
            track_idx[e] = len(lst)
            lst.append(int(model.point_ids[k]))
    cams, imgs = sorted(model.cameras.items()), sorted(model.images.items())
    p = lambda name: os.path.join(sparse_dir, f"{name}.{fmt}")   # noqa: E731
    if fmt == "txt":
        with open(p("cameras"), "w") as f:
            f.write("# CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n")
            for cid, (name, w, h, prm) in cams:
                f.write(f"{cid} {name} {w} {h} " + " ".join(repr(float(x)) for x in prm) + "\n")
        with open(p("images"), "w") as f:
            f.write("# IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME\n# POINTS2D[] as (X, Y, POINT3D_ID)\n")
            for iid, (q, t, cid, name) in imgs:
                f.write(f"{iid} " + " ".join(repr(float(x)) for x in (*q, *t)) + f" {cid} {name}\n")
                f.write(" ".join(f"0.0 0.0 {pid}" for pid in obs[iid]) + "\n")
        with open(p("points3D"), "w") as f:
            f.write("# POINT3D_ID, X, Y, Z, R, G, B, ERROR, TRACK[] as (IMAGE_ID, POINT2D_IDX)\n")
            for k in range(len(model.xyz)):
                a, b = model.track_ptr[k], model.track_ptr[k + 1]
                tr = " ".join(f"{model.track_img[e]} {track_idx[e]}" for e in range(a, b))
                f.write(f"{model.point_ids[k]} " + " ".join(repr(float(x)) for x in model.xyz[k])
                        + f" 128 128 128 0.5 {tr}\n")
        return
    with open(p("cameras"), "wb") as f:
        f.write(struct.pack("<Q", len(cams)))
        for cid, (name, w, h, prm) in cams:
            f.write(struct.pack("<iiQQ", cid, MODEL_IDS[name][0], w, h))
            f.write(struct.pack(f"<{len(prm)}d", *prm))
    with open(p("images"), "wb") as f:
        f.write(struct.pack("<Q", len(imgs)))
        for iid, (q, t, cid, name) in imgs:
            f.write(struct.pack("<i7di", iid, *q, *t, cid) + name.encode("utf-8") + b"\0")
            f.write(struct.pack("<Q", len(obs[iid])))
            f.write(b"".join(struct.pack("<ddq", 0.0, 0.0, pid) for pid in obs[iid]))
    with open(p("points3D"), "wb") as f:
        f.write(struct.pack("<Q", len(model.xyz)))
        for k in range(len(model.xyz)):
            a, b = model.track_ptr[k], model.track_ptr[k + 1]
            f.write(struct.pack("<Q3d3BdQ", model.point_ids[k], *model.xyz[k], 128, 128, 128, 0.5, b - a))
            f.write(b"".join(struct.pack("<ii", model.track_img[e], track_idx[e]) for e in range(a, b)))


# ------------------------------------------------------------------------------ scene
def qvec_to_rotmat(q):
    """COLMAP's (w, x, y, z) unit quaternion -> rotation matrix (normalised first)."""
    w, x, y, z = np.asarray(q, np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def rotmat_to_qvec(R):
    """Rotation matrix -> (w, x, y, z) unit quaternion with w >= 0 (the eigenvector of the
    symmetric 4x4 matrix built from R for its largest eigenvalue)."""
    R = np.asarray(R, np.float64).T
    K = np.array([[R[0, 0] - R[1, 1] - R[2, 2], 0, 0, 0],
                  [R[1, 0] + R[0, 1], R[1, 1] - R[0, 0] - R[2, 2], 0, 0],
                  [R[2, 0] + R[0, 2], R[2, 1] + R[1, 2], R[2, 2] - R[0, 0] - R[1, 1], 0],
                  [R[1, 2] - R[2, 1], R[2, 0] - R[0, 2], R[0, 1] - R[1, 0],
                   R[0, 0] + R[1, 1] + R[2, 2]]]) / 3.0
    w, V = np.linalg.eigh(K)
    q = V[[3, 0, 1, 2], np.argmax(w)]
    return -q if q[0] < 0 else q


def intrinsics(name, params):
    if name == "SIMPLE_PINHOLE":
        f, cx, cy = params
        fx = fy = f
    else:
        fx, fy, cx, cy = params
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])


def split_params(name, params):
    """COLMAP camera parameters -> (fx, fy, cx, cy, distortion coefficients in COLMAP's order)."""
    p = [float(x) for x in params]
    if name in SINGLE_FOCAL_MODELS:
        return p[0], p[0], p[1], p[2], p[3:]
    return p[0], p[1], p[2], p[3], p[4:]


def distortion(name, k, u, v):
    """COLMAP's forward distortion (du, dv) of normalised points (u, v) (float64 arrays) for the
    coefficients k of model `name`; the distorted pixel is (fx (u + du) + cx, fy (v + dv) + cy)."""
    k = list(k) + [0.0] * 8
    u2, v2, uv = u * u, v * v, u * v
    r2 = u2 + v2
    if name in FISHEYE_MODELS:
        r = np.sqrt(r2)
        th = np.arctan(r)
        t2 = th * th
        thd = th * ((((1.0 + k[0] * t2) + k[1] * t2 ** 2) + k[2] * t2 ** 3) + k[3] * t2 ** 4)
        rs = np.where(r > 0, r, 1.0)
        return np.where(r > 0, u * thd / rs - u, 0.0), np.where(r > 0, v * thd / rs - v, 0.0)
    if name in ("SIMPLE_RADIAL", "RADIAL"):
        rad = k[0] * r2 + k[1] * r2 * r2
        return u * rad, v * rad
    p1, p2 = k[2], k[3]
    tu, tv = 2 * p1 * uv + p2 * (r2 + 2 * u2), 2 * p2 * uv + p1 * (r2 + 2 * v2)
    if name == "OPENCV":
        rad = k[0] * r2 + k[1] * r2 * r2
        return u * rad + tu, v * rad + tv
    if name == "FULL_OPENCV":
        r4, r6 = r2 * r2, r2 * r2 * r2
        rad = (1 + k[0] * r2 + k[1] * r4 + k[4] * r6) / (1 + k[5] * r2 + k[6] * r4 + k[7] * r6)
        return u * rad + tu - u, v * rad + tv - v
    raise ValueError(f"no distortion for the {name} model")


def _undistort_normalised(name, k, ud, vd):
    """(u, v) with (u, v) + distortion(u, v) = (ud, vd): Newton's method from (ud, vd) with a
    central-difference Jacobian, at most NEWTON_ITERS steps."""
    u, v = ud.copy(), vd.copy()
    for _ in range(NEWTON_ITERS):
        du, dv = distortion(name, k, u, v)
        eu, ev = u + du - ud, v + dv - vd
        hu, hv = 1e-6 * np.maximum(1.0, np.abs(u)), 1e-6 * np.maximum(1.0, np.abs(v))
        up, um = distortion(name, k, u + hu, v), distortion(name, k, u - hu, v)
        vp, vm = distortion(name, k, u, v + hv), distortion(name, k, u, v - hv)
        a, c = 1 + (up[0] - um[0]) / (2 * hu), (up[1] - um[1]) / (2 * hu)
        b, d = (vp[0] - vm[0]) / (2 * hv), 1 + (vp[1] - vm[1]) / (2 * hv)
        det = a * d - b * c
        su, sv = (d * eu - b * ev) / det, (a * ev - c * eu) / det
        u, v = u - su, v - sv
        if np.all(np.abs(su) <= 1e-15 * np.maximum(1.0, np.abs(u))) and \
                np.all(np.abs(sv) <= 1e-15 * np.maximum(1.0, np.abs(v))):
            break
    return u, v


def undistorted_camera(cid, name, w, h, params):
    """The PINHOLE camera a distorted camera `cid` is resampled to -> (W', H', [fx, fy, cx', cy']).

    Modelled on COLMAP's undistorter with blank_pixels = 0, min_scale = 0.2, max_scale = 2: the
    pixel centres of the four borders are undistorted (Newton, float64) and mapped back with the
    camera's own fx, fy, cx, cy; sx = min((cx - max_left X) / (cx - 0.5), (min_right X - cx) /
    (W - 0.5 - cx)), sy likewise in y, each clipped to [0.2, 2]; W' = max(2, round(sx W)),
    H' = max(2, round(sy H)), cx' = cx (W' / W), cy' = cy (H' / H); fx and fy are kept.
    Raises ValueError naming the camera when a parameter is not finite, a focal length is not
    positive, the size is below 2 x 2, the principal point is not inside the pixel-centre box, a
    border pixel does not round-trip within NEWTON_TOL_PX or a ratio is not positive."""
    def refuse(why):
        raise ValueError(f"camera {cid} ({name}, {w}x{h}): {why}")
    params = np.asarray(params, np.float64)
    if not np.all(np.isfinite(params)):
        refuse("a parameter is not finite")
    fx, fy, cx, cy, k = split_params(name, params)
    if not (fx > 0 and fy > 0):
        refuse("the focal length is not positive")
    if w < 2 or h < 2:
        refuse("the size is below 2 x 2")
    if not (0.5 < cx < w - 0.5 and 0.5 < cy < h - 0.5):
        refuse(f"the principal point ({cx!r}, {cy!r}) is not inside the pixel-centre box")
    xs, ys = np.arange(w) + 0.5, np.arange(h) + 0.5
    bx = np.concatenate([np.full(h, 0.5), np.full(h, w - 0.5), xs, xs])
    by = np.concatenate([ys, ys, np.full(w, 0.5), np.full(w, h - 0.5)])
    with np.errstate(all="ignore"):                 # a diverging point ends as inf / NaN
        u, v = _undistort_normalised(name, k, (bx - cx) / fx, (by - cy) / fy)
        du, dv = distortion(name, k, u, v)
        res = np.maximum(np.abs(fx * (u + du) + cx - bx), np.abs(fy * (v + dv) + cy - by))
    if not np.all(res <= NEWTON_TOL_PX):
        i = int(np.argmax(np.where(res <= NEWTON_TOL_PX, 0, 1)))
        refuse(f"the undistortion of border pixel ({bx[i]}, {by[i]}) does not converge "
               f"(residual {res[i]:.3g} px)")
    X, Y = fx * u + cx, fy * v + cy
    left, right, top, bottom = X[:h], X[h:2 * h], Y[2 * h:2 * h + w], Y[2 * h + w:]
    ratios = ((cx - left.max()) / (cx - 0.5), (right.min() - cx) / (w - 0.5 - cx),
              (cy - top.max()) / (cy - 0.5), (bottom.min() - cy) / (h - 0.5 - cy))
    if not all(r > 0 for r in ratios):
        refuse(f"a scale ratio is not positive {tuple(float(r) for r in ratios)}")
    lo, hi = UNDISTORT_SCALES
    sx = min(max(min(ratios[0], ratios[1]), lo), hi)
    sy = min(max(min(ratios[2], ratios[3]), lo), hi)
    w2, h2 = max(2, int(np.floor(sx * w + 0.5))), max(2, int(np.floor(sy * h + 0.5)))
    return w2, h2, np.array([fx, fy, cx * (w2 / w), cy * (h2 / h)])


class Scene:
    """A validated model indexed by view id (sorted image names): names [n], K (n,3,3) and
    E (n,4,4) float64, wh (n,2) camera sizes, centres (n,3), xyz (N,3), and the tracks over view
    ids in CSR form, track_ptr (N+1,) int64 / track_img (nnz,) int32, duplicates removed.
    K and wh are the camera the depth maps are computed in: the view's own for a PINHOLE or
    SIMPLE_PINHOLE camera, else its undistorted camera (undistorted_camera).  src_cameras[v] is
    the view's camera as the model has it, (model id, w, h, params), and distorted (n,) bool marks
    the views whose images must be undistorted."""

    def __init__(self, model):
        order = sorted(model.images, key=lambda i: model.images[i][3])
        self.names = [model.images[i][3] for i in order]
        n = len(order)
        self.K, self.E = np.zeros((n, 3, 3)), np.tile(np.eye(4), (n, 1, 1))
        self.wh = np.zeros((n, 2), np.int64)
        self.src_cameras, self.distorted = [], np.zeros(n, bool)
        undistorted = {}
        for v, iid in enumerate(order):
            q, t, cid, _ = model.images[iid]
            name, w, h, params = model.cameras[cid]
            self.src_cameras.append((MODEL_IDS[name][0], w, h, np.asarray(params, np.float64)))
            if name in SUPPORTED_MODELS:
                self.K[v] = intrinsics(name, params)
                self.wh[v] = (w, h)
            else:
                if cid not in undistorted:
                    undistorted[cid] = undistorted_camera(cid, name, w, h, params)
                w2, h2, pinhole = undistorted[cid]
                self.K[v] = intrinsics("PINHOLE", pinhole)
                self.wh[v] = (w2, h2)
                self.distorted[v] = True
            self.E[v, :3, :3] = qvec_to_rotmat(q)
            self.E[v, :3, 3] = t
        self.centres = -np.einsum("nji,nj->ni", self.E[:, :3, :3], self.E[:, :3, 3])
        self.xyz = model.xyz
        ids = np.array(order, np.int64)
        by_id = np.argsort(ids)
        img = by_id[np.searchsorted(ids[by_id], model.track_img)] if n else model.track_img
        pt = np.repeat(np.arange(len(model.xyz)), np.diff(model.track_ptr))
        # one entry per (point, view): sort by (point, view) and drop repeats
        o = np.lexsort((img, pt))
        pt, img = pt[o], img[o]
        keep = np.ones(len(pt), bool)
        keep[1:] = (pt[1:] != pt[:-1]) | (img[1:] != img[:-1])
        pt, img = pt[keep], img[keep]
        self.track_img = img.astype(np.int32)
        self.track_ptr = np.zeros(len(model.xyz) + 1, np.int64)
        np.cumsum(np.bincount(pt, minlength=len(model.xyz)), out=self.track_ptr[1:])

    def __len__(self):
        return len(self.names)


def load_scene(root):
    return Scene(read_model(find_sparse_dir(root), distorted=True))


def view_scores(centres, xyz, track_ptr, track_img, device="cuda:0", max_chunk_pairs=0):
    """(n,n) float64 CUDA tensor of casmvs_view_scores_fwd.  max_chunk_pairs > 0 caps the pairs
    per chunk (smaller workspace, same bits)."""
    import ctypes

    from . import _lib
    dev = torch.device(device)
    t = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a), dtype=dt).to(dev)   # noqa: E731
    c, p = t(centres, torch.float64), t(xyz, torch.float64)
    ptr, img = t(track_ptr, torch.int64), t(track_img, torch.int32)
    n, npts = int(c.shape[0]), int(p.shape[0])
    out = torch.empty(n, n, dtype=torch.float64, device=dev)
    lib = _lib.load()
    nbytes = lib.casmvs_view_scores_workspace_bytes(n, npts, int(max_chunk_pairs))
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    vp = lambda x: ctypes.c_void_p(x.data_ptr())   # noqa: E731
    with torch.cuda.device(dev):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(lib.casmvs_view_scores_fwd(vp(c), vp(p), vp(ptr), vp(img), n, npts, vp(out),
                                              vp(ws), nbytes, st), "view_scores")
    return out


def depth_stats(E, xyz, track_ptr, track_img, device="cuda:0", quantiles=DEPTH_QUANTILES):
    """Per view: the number of its observed points with z > 0 in its camera, and q(f) for each
    f of `quantiles` over those z (NaN for a view with none) -> (count (n,) int64, q (n, len(f))
    float64), host arrays.  z, the per-view sort and the picks run as torch ops on `device`."""
    dev = torch.device(device)
    n = len(E)
    Et = torch.as_tensor(np.asarray(E, np.float64), device=dev)
    P = torch.as_tensor(np.asarray(xyz, np.float64), device=dev)
    img = torch.as_tensor(np.asarray(track_img, np.int64), device=dev)
    pt = torch.repeat_interleave(torch.arange(len(track_ptr) - 1, device=dev),
                                 torch.as_tensor(np.diff(track_ptr), device=dev))
    z = (Et[img, 2, :3] * P[pt]).sum(1) + Et[img, 2, 3]
    front = z > 0
    z, img = z[front], img[front]
    o = torch.argsort(z, stable=True)
    o = o[torch.argsort(img[o], stable=True)]
    z = z[o]
    count = torch.bincount(img, minlength=n).cpu().numpy()
    start = np.concatenate([[0], np.cumsum(count)[:-1]])
    idx = np.array([[s + int(np.floor(f * (c - 1))) for f in quantiles] for s, c in zip(start, count)],
                   np.int64).reshape(n, len(quantiles))
    q = z[torch.as_tensor(np.clip(idx, 0, max(len(z) - 1, 0)), device=dev)].cpu().numpy() \
        if len(z) else np.zeros((n, len(quantiles)))
    q[count == 0] = np.nan
    return count.astype(np.int64), q


def select_sources(scores, n_src=N_SRC):
    """For each view, the n_src views with the highest positive score, by score descending and
    view id ascending on a tie -> [[(src, score)]]."""
    s = np.asarray(scores, np.float64)
    out = []
    for v in range(len(s)):
        ids = np.arange(len(s))
        o = np.lexsort((ids, -s[v]))
        out.append([(int(j), float(s[v, j])) for j in o if j != v and s[v, j] > 0][:n_src])
    return out


def assemble(scores, count, q, n_views, n_src=N_SRC, min_front=MIN_FRONT_POINTS):
    """-> (sources [[(src, score)]] per view, refs [view ids kept as reference views],
    skipped {vid: reason}, depth_min (n,), depth_max (n,)) with the module's rules."""
    sources = select_sources(scores, n_src)
    depth_min = DEPTH_WIDEN[0] * q[:, 0]
    depth_max = DEPTH_WIDEN[1] * q[:, 1]
    refs, skipped = [], {}
    for v in range(len(sources)):
        if len(sources[v]) < n_views - 1:
            skipped[v] = f"{len(sources[v])} valid sources < n_views - 1 = {n_views - 1}"
        elif count[v] < min_front:
            skipped[v] = f"{count[v]} observed points in front < {min_front}"
        else:
            refs.append(v)
    return sources, refs, skipped, depth_min, depth_max


def cam_text(E, K, depth_min, interval, n_depths, depth_max):
    """An MVSNet cam file; every value is written so that parsing it back gives the same float."""
    fmt = lambda r: " ".join(repr(float(x)) for x in r)      # noqa: E731
    rows = ["extrinsic"] + [fmt(r) for r in E] + ["", "intrinsic"] + [fmt(r) for r in K]
    rows += ["", f"{float(depth_min)!r} {float(interval)!r} {n_depths:g} {float(depth_max)!r}"]
    return "\n".join(rows) + "\n"


def write_cams(cam_dir, E, K, depth_range, n_depths):
    """<cam_dir>/{vid:08d}_cam.txt for every view of depth_range {vid: (dmin, interval, dmax)}."""
    os.makedirs(cam_dir, exist_ok=True)
    for v, (dmin, dint, dmax) in depth_range.items():
        with open(os.path.join(cam_dir, f"{v:08d}_cam.txt"), "w") as f:
            f.write(cam_text(E[v], K[v], dmin, dint, n_depths, dmax))


def write_pair(path, metas_scored):
    """pair.txt of [(ref, [(src, score)])] in io.read_pair_file's format."""
    lines = [str(len(metas_scored))]
    for ref, srcs in metas_scored:
        lines += [str(ref), f"{len(srcs)} " + " ".join(f"{s} {sc!r}" for s, sc in srcs)]
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")


def write_view_names(path, names):
    with open(path, "w") as f:
        f.write("".join(f"{v} {name}\n" for v, name in enumerate(names)))
