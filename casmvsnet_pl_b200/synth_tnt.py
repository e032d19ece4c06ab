"""Seeded synthetic Tanks and Temples training scenes for tnt_eval.py, in the ground-truth layout

    <gt>/<Scene>/<Scene>.ply, <Scene>.json, <Scene>_trans.txt, <Scene>_COLMAP_SfM.log

make_scene writes analytic surfaces a few metres across (a ground plane, a sphere on it and a
vertical wall) as the laser scan, a Z-axis crop polygon, a known SfM -> ground-truth similarity
and a ring of SfM cameras around the object, plus a reconstruction of the same surfaces: in a
frame related to the ground truth by a known similarity (scale 0.3 .. 3), with noise, a missing
patch, outliers 5 to 20 tau off the surfaces and points outside the crop, recorded as a run (cams/*_cam.txt, view_names.txt)
whose trajectory misses a few cameras and has a few perturbed ones, and the complete image
listing (empty files) to pair them by name.

write_gt_for_colmap writes a ground-truth directory for a synth_scenes.make_colmap capture: its
analytic surface as the scan, its own cameras as the SfM log and the identity as _trans.txt.
"""
from __future__ import annotations

import os

import numpy as np

from . import colmap, fusion


def _rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    return colmap.qvec_to_rotmat(q)


def similarity(rng, scale_range=(0.3, 3.0), shift=5.0):
    T = np.eye(4)
    T[:3, :3] = rng.uniform(*scale_range) * _rotation(rng)
    T[:3, 3] = rng.uniform(-shift, shift, 3)
    return T


def _apply(T, p):
    return p @ T[:3, :3].T + T[:3, 3]


def sample_surfaces(rng, n):
    """n points on the plane z = 0 over [-2.5, 2.5]^2, a sphere of radius 0.8 at (0, 0, 0.8) and
    a wall x = -1.5, |y| < 1.5, 0 < z < 1.5, by area.  -> (points (n,3), surface id (n,))."""
    areas = np.array([25.0, 4 * np.pi * 0.64, 4.5])
    which = rng.choice(3, n, p=areas / areas.sum())
    p = np.empty((n, 3))
    k = which == 0
    p[k] = np.c_[rng.uniform(-2.5, 2.5, (k.sum(), 2)), np.zeros(k.sum())]
    k = which == 1
    d = rng.normal(size=(k.sum(), 3))
    p[k] = 0.8 * d / np.linalg.norm(d, axis=1, keepdims=True) + [0, 0, 0.8]
    k = which == 2
    p[k] = np.c_[np.full(k.sum(), -1.5), rng.uniform(-1.5, 1.5, k.sum()), rng.uniform(0, 1.5, k.sum())]
    return p, which


def surface_mesh(res=1.0):
    """The plane, sphere and wall of sample_surfaces triangulated in the ground-truth frame ->
    (verts (V,3) float64, faces (F,3) int32): grids of 100 res x 100 res squares on the plane,
    256 res x 128 res longitude-latitude cells on the sphere and 30 x 15 squares on the wall."""
    parts, faces, off = [], [], 0
    for P in _surface_grids(res):
        nv, nu = P.shape[0] - 1, P.shape[1] - 1
        i = (np.arange(nu)[None, :] + (nu + 1) * np.arange(nv)[:, None]).ravel() + off
        faces.append(np.concatenate([np.stack([i, i + 1, i + nu + 2], 1),
                                     np.stack([i, i + nu + 2, i + nu + 1], 1)]))
        parts.append(P.reshape(-1, 3))
        off += len(parts[-1])
    return np.concatenate(parts), np.concatenate(faces).astype(np.int32)


def _surface_grids(res):
    n = int(100 * res)
    u, w = np.meshgrid(np.linspace(-2.5, 2.5, n + 1), np.linspace(-2.5, 2.5, n + 1), indexing="xy")
    yield np.stack([u, w, np.zeros_like(u)], -1)
    nt, nz = int(256 * res), int(128 * res)
    th, ph = np.meshgrid(np.linspace(0, 2 * np.pi, nt + 1), np.linspace(0, np.pi, nz + 1), indexing="xy")
    yield np.stack([0.8 * np.sin(ph) * np.cos(th), 0.8 * np.sin(ph) * np.sin(th),
                    0.8 + 0.8 * np.cos(ph)], -1)
    u, w = np.meshgrid(np.linspace(-1.5, 1.5, 31), np.linspace(0, 1.5, 16), indexing="xy")
    yield np.stack([np.full_like(u, -1.5), u, w], -1)


CROP_POLYGON = [[2.0, 0.0], [1.0, 1.9], [-1.9, 1.9], [-1.9, -1.9], [1.0, -1.9]]


def _look_at_c2w(centre, target):
    z = target - centre
    z /= np.linalg.norm(z)
    x = np.cross(z, [0, 0, 1.0])
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    M = np.eye(4)
    M[:3, :3] = np.stack([x, y, z], 1)
    M[:3, 3] = centre
    return M


def _rigid(M):
    """M with its 3x3 divided by the cube root of its determinant: a camera pose mapped by a
    similarity keeps its centre and stays a rotation."""
    M = M.copy()
    M[:3, :3] /= np.cbrt(np.linalg.det(M[:3, :3]))
    return M


def write_log(path, poses):
    with open(path, "w") as f:
        for k, M in enumerate(poses):
            f.write(f"{k} {k} 0\n")
            for r in M:
                f.write(" ".join(repr(float(x)) for x in r) + "\n")


def write_trans(path, T):
    with open(path, "w") as f:
        f.write("\n".join(" ".join(repr(float(x)) for x in r) for r in T) + "\n")


def write_crop(path, axis, amin, amax, polygon_xyz):
    import json
    with open(path, "w") as f:
        json.dump(dict(axis_max=float(amax), axis_min=float(amin),
                       bounding_polygon=[[float(x) for x in p] for p in polygon_xyz],
                       class_name="SelectionPolygonVolume", orthogonal_axis="XYZ"[axis],
                       version_major=1, version_minor=0), f, indent=1)


def _write_ply(path, xyz):
    xyz = np.asarray(xyz, np.float32)
    fusion.write_ply(path, xyz, np.full((len(xyz), 3), 200, np.uint8))


def write_run_cams(run_dir, c2w, names):
    """cams/{vid:08d}_cam.txt (world -> camera) and view_names.txt of the given poses."""
    K = np.array([[500.0, 0, 320], [0, 500, 240], [0, 0, 1]])
    os.makedirs(os.path.join(run_dir, "cams"), exist_ok=True)
    for v, M in enumerate(c2w):
        E = np.linalg.inv(M)
        E[3] = [0, 0, 0, 1]
        with open(os.path.join(run_dir, "cams", f"{v:08d}_cam.txt"), "w") as f:
            f.write(colmap.cam_text(E, K, 0.5, 0.01, 192, 10.0))
    colmap.write_view_names(os.path.join(run_dir, "view_names.txt"), names)


def make_scene(root, scene="Synth", n_gt=200_000, n_rec=200_000, n_cams=40, seed=0, tau=0.05,
               noise=0.25, outliers=0.002, missing_cams=3, perturbed_cams=3, cam_noise=0.01):
    """Writes <root>/gt/<scene>/..., <root>/rec.ply, <root>/run (cams, view_names.txt) and
    <root>/images; returns a dict with the paths and the true reconstruction -> ground truth
    similarity (`rec_to_gt`).  `noise` is the reconstruction's noise in units of tau."""
    rng = np.random.default_rng(seed)
    gt_dir = os.path.join(root, "gt", scene)
    os.makedirs(gt_dir, exist_ok=True)
    gt, _ = sample_surfaces(rng, n_gt)
    _write_ply(os.path.join(gt_dir, f"{scene}.ply"), gt)
    poly = np.c_[np.array(CROP_POLYGON), np.zeros(len(CROP_POLYGON))]
    write_crop(os.path.join(gt_dir, f"{scene}.json"), 2, -0.05, 1.7, poly)
    sfm_to_gt = similarity(rng, (0.5, 2.0))
    write_trans(os.path.join(gt_dir, f"{scene}_trans.txt"), sfm_to_gt)
    ang = np.linspace(0, 2 * np.pi, n_cams, endpoint=False)
    cams_gt = [_look_at_c2w(np.array([4 * np.cos(a), 4 * np.sin(a), 1.5 + 0.3 * np.sin(3 * a)]),
                            np.array([0, 0, 0.6])) for a in ang]
    gt_to_sfm = np.linalg.inv(sfm_to_gt)
    write_log(os.path.join(gt_dir, f"{scene}_COLMAP_SfM.log"), [_rigid(gt_to_sfm @ M) for M in cams_gt])

    # reconstruction, in the ground-truth frame first
    rec, which = sample_surfaces(rng, n_rec)
    rec += rng.normal(scale=noise * tau, size=rec.shape)
    hole = (which == 1) & (rec[:, 0] > 0.3) & (rec[:, 1] > 0.3)              # a missing patch
    rec = rec[~hole]
    n_out = int(outliers * len(rec))              # 5 to 20 tau off the surface, any direction
    off = rng.normal(size=(n_out, 3))
    off *= rng.uniform(5 * tau, 20 * tau, (n_out, 1)) / np.linalg.norm(off, axis=1, keepdims=True)
    rec = np.concatenate([rec, rec[rng.integers(0, len(rec), n_out)] + off])
    rec = rec[rng.permutation(len(rec))]
    gt_to_rec = similarity(rng)
    _write_ply(os.path.join(root, "rec.ply"), _apply(gt_to_rec, rec))

    names = [f"{k:06d}.jpg" for k in range(n_cams)]
    img_dir = os.path.join(root, "images")
    os.makedirs(img_dir, exist_ok=True)
    for nm in names:
        open(os.path.join(img_dir, nm), "wb").close()
    keep = np.sort(rng.choice(n_cams, n_cams - missing_cams, replace=False))
    bad = set(rng.choice(len(keep), perturbed_cams, replace=False).tolist())
    c2w = []
    for j, k in enumerate(keep):
        M = cams_gt[k].copy()
        M[:3, 3] += rng.normal(scale=cam_noise, size=3)
        if j in bad:
            off = rng.normal(size=3)
            M[:3, 3] += off / np.linalg.norm(off)                  # 1 unit: never an inlier
        c2w.append(_rigid(gt_to_rec @ M))
    run_dir = os.path.join(root, "run")
    write_run_cams(run_dir, c2w, [names[k] for k in keep])
    return dict(gt_dir=os.path.join(root, "gt"), scene=scene, ply=os.path.join(root, "rec.ply"),
                run_dir=run_dir, images=img_dir, rec_to_gt=np.linalg.inv(gt_to_rec), tau=tau)


def write_gt_for_colmap(capture_root, gt_root, scene, depth=3.0, n_points=200_000, seed=0):
    """A ground-truth directory <gt_root>/<scene> for a synth_scenes.make_colmap capture with the
    given `depth`: its surface z = depth + 0.05 depth sin(3x/depth) cos(2y/depth) over
    |x| <= 0.5 depth, |y| <= 0.3 depth as the scan, the capture's cameras in sorted image-name
    order as the SfM log, the identity as _trans.txt and a Z-axis crop around the surface."""
    rng = np.random.default_rng(seed)
    d = os.path.join(gt_root, scene)
    os.makedirs(d, exist_ok=True)
    x = rng.uniform(-0.5, 0.5, n_points) * depth
    y = rng.uniform(-0.3, 0.3, n_points) * depth
    z = depth + 0.05 * depth * np.sin(3 * x / depth) * np.cos(2 * y / depth)
    _write_ply(os.path.join(d, f"{scene}.ply"), np.stack([x, y, z], 1))
    hx, hy = 0.45 * depth, 0.28 * depth
    poly = [[hx, hy, 0], [-hx, hy, 0], [-hx, -hy, 0], [hx, -hy, 0]]
    write_crop(os.path.join(d, f"{scene}.json"), 2, 0.9 * depth, 1.1 * depth, poly)
    write_trans(os.path.join(d, f"{scene}_trans.txt"), np.eye(4))
    sc = colmap.load_scene(capture_root)
    write_log(os.path.join(d, f"{scene}_COLMAP_SfM.log"), [np.linalg.inv(E) for E in sc.E])
    return d
