"""Seeded synthetic scans in the Tanks and Temples and BlendedMVS test layouts, for the scan
readers of eval_pipeline, and in the DTU and BlendedMVS training layouts (make_dtu_train,
make_blendedmvs_train), for train_data and the trainer (the real data sets are large and
licensed separately).

  tanks       <root>/<split>/<scan>/pair.txt, cams/{vid:08d}_cam.txt, images/{vid:08d}.jpg
  blendedmvs  <root>/dataset_low_res/<scan>/cams/pair.txt, cams/{vid:08d}_cam.txt,
              blended_images/{vid:08d}.jpg, rendered_depth_maps/{vid:08d}.pfm;
              <root>/{training,validation,all}_list.txt

Cameras sit on an arc around a point ~`depth` in front of them and look at it, with full-resolution
intrinsics of the data set's native size in the cam files (tanks.py:86-87, blendedmvs.py:73-74
scale them to img_wh).  Images are blurred noise JPEGs of any size (`image_wh`: small for tests,
the native size for timing); each view's source list holds its neighbours on the arc.  With
`n_few`, every n_few-th BlendedMVS reference view lists only 2 valid sources, so readers with
n_views > 2 skip it (blendedmvs.py:51-54), and is no other view's source.

make_colmap writes the same arc of cameras as an undistorted COLMAP workspace (images/ and a
sparse/ model of points on a known surface, binary and / or text) for eval_pipeline's colmap
reader, or with distorted cameras and / or as a `colmap mapper` project (sparse/0); sparse_tracks
makes bare sparse models of any size for the view-selection kernel.
sphere_scene renders analytic depth maps and colours of a sphere (on a plane) for meshing.

    python -m casmvsnet_pl_b200.synth_scenes --kind tanks --root TNT --n_views 150 --image_wh 1920 1080
"""
from __future__ import annotations

import argparse
import os

import numpy as np
import torch

from . import io

NATIVE = {"tanks": (1920, 1080), "blendedmvs": (768, 576)}


def _cam_text(K, E, depth_min, interval):
    rows = ["extrinsic"] + [" ".join(f"{v:.6f}" for v in r) for r in E] + ["", "intrinsic"]
    rows += [" ".join(f"{v:.6f}" for v in r) for r in K] + ["", f"{depth_min} {interval}"]
    return "\n".join(rows) + "\n"


def _image(rng, w, h):
    import cv2
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    return cv2.GaussianBlur(img, (0, 0), 1.5)


def _write_views(d, n, native_wh, image_wh, depth, seed, img_dir, n_few=0, n_src=6):
    """cams/, <img_dir>/, pair.txt under d; returns the per-view depth_min."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    W, H = native_wh
    K = np.array([[1.1 * W, 0, W / 2], [0, 1.1 * W, H / 2], [0, 0, 1.0]])
    os.makedirs(os.path.join(d, "cams"), exist_ok=True)
    os.makedirs(os.path.join(d, img_dir), exist_ok=True)
    dmins = []
    for vid in range(n):
        t = np.deg2rad(2.0 * (vid - n / 2))
        E = np.eye(4)
        E[:3, :3] = [[np.cos(t), 0, np.sin(t)], [0, 1, 0], [-np.sin(t), 0, np.cos(t)]]
        E[:3, 3] = [-depth * np.sin(t), 0, depth * (1 - np.cos(t))]
        dmin = round(0.8 * depth + 0.01 * depth * rng.random(), 4)
        dmins.append(dmin)
        with open(os.path.join(d, "cams", f"{vid:08d}_cam.txt"), "w") as f:
            f.write(_cam_text(K, E, dmin, round(depth / 400, 6)))
        Image.fromarray(_image(rng, *image_wh)).save(os.path.join(d, img_dir, f"{vid:08d}.jpg"),
                                                     quality=92)
    few = {v for v in range(n) if n_few and v % n_few == n_few - 1}
    lines = [str(n)]
    for vid in range(n):
        # the views with few sources are nobody's source, so the other views keep their depth maps
        # usable in fusion (a missing source depth skips a reference view, eval.py:319-330)
        src = sorted((v for v in range(n) if v != vid and v not in few),
                     key=lambda v: (abs(v - vid), v))[:n_src]
        if vid in few:
            src = src[:2]
        lines += [str(vid), f"{len(src)} " + " ".join(f"{v} {100.0 - abs(v - vid):.1f}" for v in src)]
    with open(os.path.join(d, "pair.txt" if img_dir == "images" else os.path.join("cams", "pair.txt")),
              "w") as f:
        f.write("\n".join(lines) + "\n")
    return dmins


def make_tanks(root, split="intermediate", scan="Family", n_views=8, image_wh=(200, 120),
               depth=3.0, seed=0):
    """A Tanks-layout scan (native size from the reference's per-scan table); returns its dir."""
    from .eval_pipeline import TanksTestScan
    native = TanksTestScan.SCANS[split][scan][0]
    d = os.path.join(root, split, scan)
    _write_views(d, n_views, native, image_wh, depth, seed, "images")
    return d


def make_blendedmvs(root, scan="5a3ca9cb270f0e3f14d0eddb", n_views=8, image_wh=(192, 144),
                    depth=30.0, seed=0, n_few=4, lists=("all", "val")):
    """A BlendedMVS-layout scan under <root>/dataset_low_res (native 768x576) with rendered
    depth maps at the image size; appends the scan to the given scan lists.  Returns the
    dataset_low_res directory (the reader's root_dir)."""
    base = os.path.join(root, "dataset_low_res")
    d = os.path.join(base, scan)
    dmins = _write_views(d, n_views, NATIVE["blendedmvs"], image_wh, depth, seed, "blended_images",
                         n_few=n_few)
    rng = np.random.default_rng(seed + 1)
    os.makedirs(os.path.join(d, "rendered_depth_maps"), exist_ok=True)
    w, h = image_wh
    yy, xx = np.mgrid[:h, :w]
    for vid, dmin in enumerate(dmins):
        dep = dmin * (1.1 + 0.2 * np.sin(xx / w * 3 + vid) * np.cos(yy / h * 2)) \
            + rng.normal(0, 0.01 * dmin, (h, w))
        dep[: h // 10] = 0                                     # no rendered surface (sky)
        io.save_pfm(os.path.join(d, "rendered_depth_maps", f"{vid:08d}.pfm"), dep.astype(np.float32))
    names = {"train": "training_list.txt", "val": "validation_list.txt", "all": "all_list.txt"}
    for split in lists:
        with open(os.path.join(root, names[split]), "a") as f:
            f.write(scan + "\n")
    return base


BLENDEDMVS_TRAIN_SCANS = ("5a0000000000000000000a01", "5a0000000000000000000b02")


def make_blendedmvs_train(root, n_views=(8, 6), image_wh=(96, 72), seed=0, n_few=4):
    """Two BlendedMVS-layout scans for the training reader: BLENDEDMVS_TRAIN_SCANS[0] with
    n_views[0] views in training_list.txt and [1] with n_views[1] views in
    validation_list.txt, both in all_list.txt.  The scans differ in scene depth (30 and 45) and
    texture; every n_few-th view has too few sources and is skipped by readers with n_views > 2,
    and the top tenth of every depth map is 0 (sky).  Returns the dataset_low_res directory."""
    train, val = BLENDEDMVS_TRAIN_SCANS
    make_blendedmvs(root, train, n_views[0], tuple(image_wh), 30.0, seed, n_few, ("train", "all"))
    return make_blendedmvs(root, val, n_views[1], tuple(image_wh), 45.0, seed + 10, n_few, ("val", "all"))


def make_dtu_train(root, scan="scan1", refs=(0, 1, 2), n_src=5, depth=650.0, seed=0):
    """A scan in the DTU training layout datasets/dtu.py reads with img_wh=None:

        <root>/Cameras/pair.txt                    the viewpoints `refs`, n_src sources each
        <root>/Cameras/train/{vid:08d}_cam.txt     all 49 views (the reader loads every one)
        <root>/Rectified/<scan>_train/rect_{vid+1:03d}_{light}_r5000.png   640x512, lights 0-6
        <root>/Depths/<scan>/depth_map_{vid:04d}.pfm, depth_visual_{vid:04d}.png   1600x1200
        <root>/lists/{train,val}.txt               the scan lists (one scan per line)

    Cam files hold the intrinsics of the 160x128 coarsest level, depth_min 425 and interval
    2.65 as DTU's do.  Each light scales and shifts the view's texture differently.  Depth maps
    (about `depth` mm) and masks exist for the reference views only; masks have holes and grey
    levels other than 255.  Returns the root."""
    import cv2
    from PIL import Image
    rng = np.random.default_rng(seed)
    K = np.array([[1.1 * 160, 0, 80.0], [0, 1.1 * 160, 64.0], [0, 0, 1.0]])
    os.makedirs(os.path.join(root, "Cameras", "train"), exist_ok=True)
    for vid in range(49):
        t = np.deg2rad(1.5 * (vid - 3))
        E = np.eye(4)
        E[:3, :3] = [[np.cos(t), 0, np.sin(t)], [0, 1, 0], [-np.sin(t), 0, np.cos(t)]]
        E[:3, 3] = [-depth * np.sin(t), 0, depth * (1 - np.cos(t))]
        with open(os.path.join(root, "Cameras", "train", f"{vid:08d}_cam.txt"), "w") as f:
            f.write(_cam_text(K, E, 425.0, 2.65))
    pairs = {r: sorted((v for v in range(49) if v != r), key=lambda v: (abs(v - r), v))[:n_src]
             for r in refs}
    lines = [str(len(refs))]
    for r in refs:
        lines += [str(r), f"{n_src} " + " ".join(f"{v} {100.0 - abs(v - r):.1f}" for v in pairs[r])]
    with open(os.path.join(root, "Cameras", "pair.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    img_dir = os.path.join(root, "Rectified", f"{scan}_train")
    os.makedirs(img_dir, exist_ok=True)
    for vid in sorted(set(refs) | {v for s in pairs.values() for v in s}):
        base = _image(rng, 640, 512).astype(np.float32)
        for light in range(7):
            img = np.clip(base * (0.55 + 0.08 * light) + 6 * light - 10, 0, 255).astype(np.uint8)
            Image.fromarray(img).save(os.path.join(img_dir, f"rect_{vid + 1:03d}_{light}_r5000.png"))
    ddir = os.path.join(root, "Depths", scan)
    os.makedirs(ddir, exist_ok=True)
    yy, xx = np.mgrid[:1200, :1600]
    for vid in refs:
        dep = depth * (1 + 0.15 * np.sin(xx / 1600 * 4 + vid) * np.cos(yy / 1200 * 3)) \
            + rng.normal(0, 0.5, (1200, 1600))
        valid = (np.sin(xx / 97.0 + vid) + np.cos(yy / 61.0) > -1.2) & (rng.random((1200, 1600)) > 0.05)
        dep = np.where(valid, dep, 0).astype(np.float32)
        io.save_pfm(os.path.join(ddir, f"depth_map_{vid:04d}.pfm"), dep)
        vis = np.where(valid, rng.integers(1, 256, (1200, 1600)), 0).astype(np.uint8)
        cv2.imwrite(os.path.join(ddir, f"depth_visual_{vid:04d}.png"), vis)
    os.makedirs(os.path.join(root, "lists"), exist_ok=True)
    for split in ("train", "val"):
        with open(os.path.join(root, "lists", f"{split}.txt"), "w") as f:
            f.write(scan + "\n")
    return root


def _distorted(cam, model, coeffs):
    """A PINHOLE / SIMPLE_PINHOLE camera as `model` with the same fx, fy, cx, cy and `coeffs`."""
    from . import colmap
    name, w, h, prm = cam
    fx, fy, cx, cy, _ = colmap.split_params(name, prm)
    single = model in colmap.SINGLE_FOCAL_MODELS
    if single and fx != fy:
        raise ValueError(f"{model} has one focal length; the {name} camera has fx {fx} != fy {fy}")
    params = ([fx] if single else [fx, fy]) + [cx, cy] + [float(c) for c in coeffs]
    if len(params) != colmap.MODEL_IDS[model][1]:
        raise ValueError(f"{model} takes {colmap.MODEL_IDS[model][1] - (3 if single else 4)} "
                         f"coefficients, got {len(coeffs)}")
    return (model, w, h, np.array(params))


def colmap_model(n_views=8, image_wh=(160, 120), depth=3.0, n_points=2000, seed=0, n_single=20,
                 n_dup=20, distortion=None, ext="jpg", tilt=0.0):
    """The arc cameras of the other layouts as a COLMAP model (colmap.ColmapModel) looking at a
    known surface, z = depth + 0.05 depth sin(3x / depth) cos(2y / depth) in world coordinates,
    which every optical axis meets at depth `depth` (the cameras sit on a circle of that radius
    around (0, 0, depth) and look at its centre).  Even views use a PINHOLE camera of `image_wh`,
    odd views a SIMPLE_PINHOLE camera 1.25 times larger.  Image ids are shuffled against the
    sorted image names.  A point's track is every view it projects into with z > 0; the first
    n_single tracks of length > 1 are cut to one view and n_dup others list their first view
    twice.  `distortion`, (model, coefficients) or {camera id: (model, coefficients)}, turns
    both cameras (or the ones named) into that COLMAP model with the same fx, fy, cx and cy
    (tracks as without it); `ext` is the image names' extension.
    tilt != 0 adds tilt*y to the surface's z: a slope that recedes towards the bottom of every
    image (tilt > 0), so one view sees a wide range of depths (tilt 2.25 at the default focal
    length: about 0.55 to 5.5 times `depth` from the top row to the bottom one); the points then
    cover y in [-0.3, 2.2] * depth.  tilt = 0 gives the model it always gave."""
    from . import colmap
    rng = np.random.default_rng(seed)
    W, H = image_wh
    W2, H2 = int(round(W * 1.25)), int(round(H * 1.25))
    cams = {1: ("PINHOLE", W, H, np.array([1.1 * W, 1.1 * W * 1.01, W / 2, H / 2])),
            2: ("SIMPLE_PINHOLE", W2, H2, np.array([1.1 * W2, W2 / 2, H2 / 2]))}
    ids = rng.permutation(n_views) + 1
    images, Es, Ks, whs = {}, [], [], []
    for v in range(n_views):
        t = np.deg2rad(2.0 * (v - n_views / 2))
        R = np.array([[np.cos(t), 0, np.sin(t)], [0, 1, 0], [-np.sin(t), 0, np.cos(t)]])
        tv = np.array([-depth * np.sin(t), 0, depth * (1 - np.cos(t))])
        cid = 1 if v % 2 == 0 else 2
        images[int(ids[v])] = (colmap.rotmat_to_qvec(R), tv, cid, f"view_{v:03d}.{ext}")
        E = np.eye(4)
        E[:3, :3], E[:3, 3] = R, tv
        name, w, h, prm = cams[cid]
        Es.append(E)
        Ks.append(colmap.intrinsics(name, prm))
        whs.append((w, h))
    x = rng.uniform(-0.5, 0.5, n_points) * depth
    y = rng.uniform(-0.3, 0.3, n_points) * depth if tilt == 0 else \
        rng.uniform(-0.3, 2.2, n_points) * depth
    xyz = np.stack([x, y, depth + tilt * y + 0.05 * depth * np.sin(3 * x / depth) * np.cos(2 * y / depth)], 1)
    tracks = []
    for p in xyz:
        tr = []
        for v in range(n_views):
            q = Ks[v] @ (Es[v][:3, :3] @ p + Es[v][:3, 3])
            if q[2] > 0 and 0 <= q[0] / q[2] < whs[v][0] and 0 <= q[1] / q[2] < whs[v][1]:
                tr.append(int(ids[v]))
        tracks.append(tr)
    long_ = [k for k, tr in enumerate(tracks) if len(tr) > 1]
    for k in long_[:n_single]:
        tracks[k] = tracks[k][:1]
    for k in long_[n_single:n_single + n_dup]:
        tracks[k] = tracks[k] + tracks[k][:1]
    keep = [k for k, tr in enumerate(tracks) if tr]
    ptr = np.zeros(len(keep) + 1, np.int64)
    np.cumsum([len(tracks[k]) for k in keep], out=ptr[1:])
    img = np.array([i for k in keep for i in tracks[k]], np.int64)
    if distortion is not None:
        per_cam = distortion if isinstance(distortion, dict) else {cid: distortion for cid in cams}
        for cid, (model, coeffs) in per_cam.items():
            cams[cid] = _distorted(cams[cid], model, coeffs)
    return colmap.ColmapModel(cams, images, 1 + 3 * np.arange(len(keep)), xyz[keep], ptr, img)


def sparse_tracks(n_img=300, n_pts=500_000, track_len=(3, 11), seed=0):
    """A seeded sparse reconstruction for view selection alone, as arrays: centres (n_img,3) on
    a circle of radius 10 around the origin, points (n_pts,3) near the origin, and tracks in CSR
    form (track_ptr (n_pts+1,) int64, track_img int32) of distinct images, lengths uniform in
    track_len (inclusive), each a random subset of a window of neighbouring images.  The
    defaults are the size of a Tanks and Temples scene (mean track 7)."""
    rng = np.random.default_rng(seed)
    a = np.linspace(0, 2 * np.pi, n_img, endpoint=False)
    centres = np.stack([10 * np.cos(a), 10 * np.sin(a), rng.uniform(-1, 1, n_img)], 1)
    xyz = rng.normal(0, 2, (n_pts, 3))
    lens = rng.integers(track_len[0], track_len[1] + 1, n_pts)
    ptr = np.zeros(n_pts + 1, np.int64)
    np.cumsum(lens, out=ptr[1:])
    win = min(n_img, max(2 * track_len[1], 16))
    img = np.empty(ptr[-1], np.int32)
    first = rng.integers(0, n_img, n_pts)
    for L in np.unique(lens):
        sel = np.nonzero(lens == L)[0]
        pick = np.argsort(rng.random((len(sel), win)), 1)[:, :L]    # L distinct offsets per point
        img[(ptr[sel][:, None] + np.arange(L)).ravel()] = ((first[sel][:, None] + pick) % n_img).ravel()
    return centres, xyz, ptr, img


def height_field_depth(K, E, wh, depth=3.0, tilt=0.0):
    """Per-pixel depth (h,w) float64 of colmap_model's surface z = depth + 0.05 depth
    sin(3x / depth) cos(2y / depth) seen by a pinhole camera K (3,3), world->camera E (4,4) of
    size wh = (w, h): the camera z of the ray-surface intersection through each pixel centre,
    found by Newton's method in float64 (the surface's slope is at most 0.15, so from the
    plane z = depth it converges in a few steps).  tilt: colmap_model's tilt, the surface then
    starts from the plane z = depth + tilt*y.  Also returns the world points (h,w,3)."""
    w, h = wh
    K, E = np.asarray(K, np.float64), np.asarray(E, np.float64)
    R, t = E[:3, :3], E[:3, 3]
    C = -R.T @ t
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    r = np.einsum("ij,hwj->hwi", R.T @ np.linalg.inv(K), np.stack([xs, ys, np.ones_like(xs)], -1))
    a, b = 3.0 / depth, 2.0 / depth
    s = (depth - C[2] + tilt * C[1]) / (r[..., 2] - tilt * r[..., 1])
    for _ in range(50):
        X = C + s[..., None] * r
        hz = depth + tilt * X[..., 1] + 0.05 * depth * np.sin(a * X[..., 0]) * np.cos(b * X[..., 1])
        dhx = 0.05 * depth * a * np.cos(a * X[..., 0]) * np.cos(b * X[..., 1])
        dhy = tilt - 0.05 * depth * b * np.sin(a * X[..., 0]) * np.sin(b * X[..., 1])
        g = X[..., 2] - hz
        step = g / (r[..., 2] - dhx * r[..., 0] - dhy * r[..., 1])
        s = s - step
        if np.abs(step).max() < 1e-13 * depth:
            break
    X = C + s[..., None] * r
    return s, X


def surface_texture(X, seed, px_per_unit):
    """A seeded band-limited RGB texture (h,w,3) uint8 at world points X (h,w,3): 16 plane waves
    in world (x, y) per channel, their periods between 16 and 64 pixels at `px_per_unit` image
    pixels per world unit, so even the strided quarter-resolution level sees them unaliased."""
    rng = np.random.default_rng(seed)
    out = np.empty(X.shape[:2] + (3,))
    for c in range(3):
        acc = np.zeros(X.shape[:2])
        for _ in range(16):
            f = px_per_unit / rng.uniform(16, 64)
            th = rng.uniform(0, 2 * np.pi)
            acc += np.sin(2 * np.pi * f * (np.cos(th) * X[..., 0] + np.sin(th) * X[..., 1])
                          + rng.uniform(0, 2 * np.pi))
        out[..., c] = 0.5 + 0.4 * acc / 16 * 2.5
    return np.clip(np.rint(out * 255), 0, 255).astype(np.uint8)


def make_colmap(root, n_views=8, image_wh=(160, 120), depth=3.0, n_points=2000, seed=0,
                fmt="bin", layout="undistorted", image_ext="jpg", image_dir=None, textured=False, **kw):
    """An undistorted COLMAP workspace: <root>/images/view_XXX.jpg at each view's camera size and
    the model of colmap_model under <root>/sparse, in binary ("bin"), text ("txt") or both
    formats ("both"; the reader prefers the binary one).  layout="mapper" puts the model under
    <root>/sparse/0 as `colmap mapper` does; image_ext="png" writes lossless images (the same
    bytes from every decoder); image_dir replaces <root>/images; `distortion` (colmap_model)
    makes the cameras distorted.  Returns the model.

    textured=True instead renders every view of the model's surface with one seeded texture in
    world coordinates (surface_texture), always as lossless PNGs, so the views agree
    photometrically under the true depth; it returns (model, depths) with depths[v] the (h,w)
    float64 ground-truth depth of view v (height_field_depth) at its camera's size."""
    from PIL import Image

    from . import colmap
    if layout not in ("undistorted", "mapper") or image_ext not in ("jpg", "png"):
        raise ValueError(f"unknown layout {layout!r} or image extension {image_ext!r}")
    if textured:
        if kw.get("distortion") is not None:
            raise ValueError("textured views are rendered with pinhole cameras; no distortion")
        image_ext = "png"
    tilt = kw.get("tilt", 0.0)
    model = colmap_model(n_views, image_wh, depth, n_points, seed, ext=image_ext, **kw)
    rng = np.random.default_rng(seed + 1)
    image_dir = image_dir or os.path.join(root, "images")
    os.makedirs(image_dir, exist_ok=True)
    depths = {}
    for q, t, cid, name in model.images.values():
        cam_name, w, h, prm = model.cameras[cid]
        opts = {"quality": 92} if image_ext == "jpg" else {}
        if textured:
            E = np.eye(4)
            E[:3, :3], E[:3, 3] = colmap.qvec_to_rotmat(q), t
            K = colmap.intrinsics(cam_name, prm)
            v = int(name[len("view_"):-len(".png")])
            depths[v], X = height_field_depth(K, E, (w, h), depth, tilt)
            img = surface_texture(X, seed + 1, K[0, 0] / depth)
        else:
            img = _image(rng, w, h)
        Image.fromarray(img).save(os.path.join(image_dir, name), **opts)
    sparse = os.path.join(root, "sparse", "0") if layout == "mapper" else os.path.join(root, "sparse")
    for f in (("bin", "txt") if fmt == "both" else (fmt,)):
        colmap.write_model(sparse, model, f)
    if textured:
        return model, [depths[v] for v in range(n_views)]
    return model


def _look_at(centre, target):
    """World -> camera rotation (rows x, y, z) of a camera at `centre` looking at `target`, image
    y pointing down (world z up)."""
    z = target - centre
    z /= np.linalg.norm(z)
    up = np.array([0.0, 0.0, 1.0]) if abs(z[2]) < 0.99 else np.array([0.0, 1.0, 0.0])
    x = np.cross(-up, z)
    x /= np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z])


def sphere_scene(n_views, image_wh, seed=0, radius=1.0, plane=True, device="cpu"):
    """Analytic depth maps for meshing: a sphere of `radius` at the origin, resting on the square
    |x|, |y| <= 3 radius of the plane z = -radius when `plane`.  With the plane, the cameras sit on
    the upper hemisphere (elevation 15..60 degrees), else all around (a Fibonacci sphere), 3.5 to
    4.5 radii from the origin, aimed at a point near it (seeded jitter).  f = 0.9 W, principal
    point at the image centre.  Pixels that see nothing have depth 0.  Returns a list of dicts
    per view: depth (H,W) float32 (z-depth), image (H,W,3) float32 colours 0..255 from the surface
    position, P (4,4) float32 numpy world -> pixel, points (N,3) float32 of the pixels with depth;
    tensors on `device` (computed in float64)."""
    rng = np.random.default_rng(seed)
    W, H = image_wh
    K = np.array([[0.9 * W, 0, W / 2], [0, 0.9 * W, H / 2], [0, 0, 1]], dtype=np.float64)
    f64 = dict(dtype=torch.float64, device=device)
    ys, xs = torch.meshgrid(torch.arange(H, **f64), torch.arange(W, **f64), indexing="ij")
    rays_cam = torch.stack([(xs - K[0, 2]) / K[0, 0], (ys - K[1, 2]) / K[1, 1], torch.ones_like(xs)], -1)
    views = []
    for i in range(n_views):
        if plane:
            el, az = np.radians(rng.uniform(15, 60)), 2 * np.pi * (i + rng.uniform(0, 0.5)) / n_views
        else:                                   # Fibonacci sphere
            el = np.arcsin(1 - 2 * (i + 0.5) / n_views)
            az = i * np.pi * (3 - np.sqrt(5)) + rng.uniform(0, 0.1)
        dist = radius * rng.uniform(3.5, 4.5)
        C = dist * np.array([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)])
        R = _look_at(C, rng.uniform(-0.1, 0.1, 3) * radius)
        d = rays_cam @ torch.as_tensor(R, **f64)         # world directions, camera z component 1
        o = torch.as_tensor(C, **f64)
        # sphere: |o + s d|^2 = r^2, nearest root
        a, b, c = (d * d).sum(-1), 2 * (d @ o), float(o @ o) - radius ** 2
        disc = b * b - 4 * a * c
        s_sph = torch.where(disc >= 0, (-b - torch.sqrt(disc.clamp(min=0))) / (2 * a), torch.inf)
        s_sph = torch.where(s_sph > 0, s_sph, torch.inf)
        s = s_sph
        if plane:
            s_pl = (-radius - o[2]) / d[..., 2]
            p = o + s_pl[..., None] * d
            ok = (s_pl > 0) & (p[..., 0].abs() <= 3 * radius) & (p[..., 1].abs() <= 3 * radius)
            s = torch.minimum(s, torch.where(ok, s_pl, torch.inf))
        hit = torch.isfinite(s)
        X = o + torch.where(hit, s, 0.0)[..., None] * d
        on_sph = hit & (s == s_sph)
        u = X / radius
        check = ((torch.floor(2 * u[..., 0]) + torch.floor(2 * u[..., 1])) % 2) * 120 + 60
        rgb = torch.stack([torch.where(on_sph, 128 + 100 * u[..., 0], check),
                           torch.where(on_sph, 128 + 100 * u[..., 1], check),
                           torch.where(on_sph, 128 + 100 * u[..., 2], 0.5 * check)], -1)
        P = np.eye(4)
        P[:3, :3], P[:3, 3] = K @ R, K @ (-R @ C)
        views.append(dict(depth=torch.where(hit, s, 0.0).float(),
                          image=torch.where(hit[..., None], rgb, 0.0).float(),
                          P=P.astype(np.float32), points=X[hit].float()))
    return views


def main(argv=None):
    ap = argparse.ArgumentParser(description="Write a seeded synthetic Tanks / BlendedMVS scan.")
    ap.add_argument("--kind", choices=["tanks", "blendedmvs"], required=True)
    ap.add_argument("--root", required=True)
    ap.add_argument("--scan", default=None)
    ap.add_argument("--n_views", type=int, default=8)
    ap.add_argument("--image_wh", nargs=2, type=int, default=None)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    if a.kind == "tanks":
        make_tanks(a.root, scan=a.scan or "Family", n_views=a.n_views,
                   image_wh=tuple(a.image_wh or (200, 120)), seed=a.seed)
    else:
        make_blendedmvs(a.root, scan=a.scan or "5a3ca9cb270f0e3f14d0eddb", n_views=a.n_views,
                        image_wh=tuple(a.image_wh or (192, 144)), seed=a.seed)


if __name__ == "__main__":
    main()
