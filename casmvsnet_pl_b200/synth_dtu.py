"""Seeded synthetic DTU-like scenes for the point-cloud scorer (dtu_eval): real DTU ground truth
is large and licensed separately, so the tests and the timing runs generate their own.

A scene is a smooth height field (a DTU-sized object when n_stl is ~3M) sampled at the STL density
of ~25 points / mm^2 (0.2 mm spacing), with:

  STL              <gt>/Points/stl/stl{NNN}_total.ply    surface samples
  ObsMask, BB, Res <gt>/ObsMask/ObsMask{N}_10.mat        BB = STL bounds +- 10 mm, Res = 1 mm,
                                                         mask = voxels within 3 mm of the STL
  P                <gt>/ObsMask/Plane{N}.mat             a ground plane below most of the surface
  data             (N,3) float32, optionally <ply_dir>/scan{N}.ply: surface samples with Gaussian
                   noise, a disc of the surface left out (a region the reconstruction missed),
                   exact duplicates and outliers out to ~100 mm beyond BB

    python -m casmvsnet_pl_b200.synth_dtu --gt_dir GT --ply_dir PLY --n_stl 3000000 --n_data 8000000
"""
from __future__ import annotations

import argparse
import os

import numpy as np

STL_DENSITY = 25.0          # points per mm^2: 0.2 mm spacing
CENTER = np.array([20.0, -30.0, 600.0])


def _height(x, y, L):
    """Surface z(x, y) over [-L/2, L/2]^2 relative to CENTER."""
    return 0.08 * L * np.sin(2 * np.pi * x / L) * np.cos(2 * np.pi * y / L) + 0.05 * L * np.cos(
        np.pi * x / L)


def _surface(rng, n, L):
    x = rng.uniform(-L / 2, L / 2, n)
    y = rng.uniform(-L / 2, L / 2, n)
    return np.stack([x, y, _height(x, y, L)], axis=1)


def height_mesh(stl, step, shift=0.0):
    """The scene's height field triangulated over the x, y extent of its STL points `stl` (N,3)
    on a grid of about `step` mm, lifted by `shift` mm in z -> (verts (V,3) float32, faces (F,3)
    int32, L, the grid cells' diagonal)."""
    L = float(np.sqrt(len(stl) / STL_DENSITY))
    lo = np.asarray(stl, np.float64)[:, :2].min(0) - CENTER[:2]
    hi = np.asarray(stl, np.float64)[:, :2].max(0) - CENTER[:2]
    m = [int(np.ceil((hi[k] - lo[k]) / step)) for k in range(2)]
    x, y = np.meshgrid(np.linspace(lo[0], hi[0], m[0] + 1), np.linspace(lo[1], hi[1], m[1] + 1),
                       indexing="xy")
    z = _height(x, y, L) + shift
    verts = (np.stack([x.ravel(), y.ravel(), z.ravel()], 1) + CENTER).astype(np.float32)
    i = (np.arange(m[0])[None, :] + (m[0] + 1) * np.arange(m[1])[:, None]).ravel()
    faces = np.concatenate([np.stack([i, i + 1, i + m[0] + 2], 1),
                            np.stack([i, i + m[0] + 2, i + m[0] + 1], 1)]).astype(np.int32)
    return verts, faces, L, float(np.hypot(*[(hi[k] - lo[k]) / m[k] for k in range(2)]))


def write_ground_truth(gt_dir, scan, stl, ground_z, empty_mask=False, res=1.0):
    """Writes the DTU ground-truth layout for the STL cloud `stl` (N,3): BB = bounds +- 10 mm,
    ObsMask = voxels of edge `res` within 3 voxels of an STL point (all false with empty_mask),
    ground plane z = ground_z.  Returns BB (2,3)."""
    import scipy.io
    import scipy.ndimage

    from .fusion import write_ply
    stl = np.asarray(stl, np.float32)
    s64 = stl.astype(np.float64)
    bb = np.stack([s64.min(0) - 10.0, s64.max(0) + 10.0])
    dims = np.floor((bb[1] - bb[0]) / res).astype(int) + 1
    mask = np.zeros(dims, dtype=bool)
    if not empty_mask:
        v = np.floor((s64 - bb[0]) / res + 0.5).astype(int)
        mask[v[:, 0], v[:, 1], v[:, 2]] = True
        mask = scipy.ndimage.binary_dilation(mask, iterations=3)
    os.makedirs(os.path.join(gt_dir, "Points", "stl"), exist_ok=True)
    os.makedirs(os.path.join(gt_dir, "ObsMask"), exist_ok=True)
    write_ply(os.path.join(gt_dir, "Points", "stl", f"stl{scan:03d}_total.ply"), stl,
              np.full((len(stl), 3), 128, np.uint8))
    scipy.io.savemat(os.path.join(gt_dir, "ObsMask", f"ObsMask{scan}_10.mat"),
                     {"ObsMask": mask, "BB": bb, "Res": np.array([[res]])})
    scipy.io.savemat(os.path.join(gt_dir, "ObsMask", f"Plane{scan}.mat"),
                     {"P": np.array([[0.0], [0.0], [1.0], [-float(ground_z)]])})
    return bb


def make_scene(gt_dir, scan=1, n_stl=100_000, n_data=200_000, seed=0, ply_dir=None,
               noise=0.15, dup_frac=0.05, outlier_frac=0.02, hole_frac=0.1, empty_mask=False):
    """Writes the ground-truth layout of scan `scan` under gt_dir (and scan{N}.ply under ply_dir if
    given); returns the data cloud (n_data, 3) float32."""
    from .fusion import write_ply
    rng = np.random.default_rng(seed)
    L = float(np.sqrt(max(n_stl, 1) / STL_DENSITY))
    stl = _surface(rng, n_stl, L) + CENTER
    stl32 = stl.astype(np.float32)

    z0 = CENTER[2] - 0.08 * L                  # ground plane z = z0: most of the surface above it
    # data: noisy samples of the surface outside a missed disc, duplicates, outliers
    n_out = int(n_data * outlier_frac)
    n_dup = int(n_data * dup_frac)
    n_surf = n_data - n_out - n_dup
    surf = np.zeros((0, 3))
    hole_r = np.sqrt(hole_frac * L * L / np.pi)
    hole_c = np.array([0.25 * L, -0.2 * L])
    while len(surf) < n_surf:
        s = _surface(rng, int((n_surf - len(surf)) * (1 + hole_frac) + 16), L)
        s = s[((s[:, :2] - hole_c) ** 2).sum(1) > hole_r ** 2]
        surf = np.concatenate([surf, s])[:n_surf]
    surf = surf + CENTER + rng.normal(0.0, noise, surf.shape)
    bb = np.stack([stl.min(0) - 10.0, stl.max(0) + 10.0])
    outl = rng.uniform(bb[0] - 100.0, bb[1] + 100.0, (n_out, 3))
    data = np.concatenate([surf, outl]).astype(np.float32)
    dups = data[rng.integers(0, max(len(data), 1), n_dup)] if len(data) else np.zeros((0, 3), np.float32)
    data = np.concatenate([data, dups])
    data = data[rng.permutation(len(data))]

    write_ground_truth(gt_dir, scan, stl32, z0, empty_mask)
    if ply_dir:
        os.makedirs(ply_dir, exist_ok=True)
        write_ply(os.path.join(ply_dir, f"scan{scan}.ply"), data, np.zeros((len(data), 3), np.uint8))
    return data


def main(argv=None):
    ap = argparse.ArgumentParser(description="Write a seeded synthetic DTU-like scene.")
    ap.add_argument("--gt_dir", required=True)
    ap.add_argument("--ply_dir", default="")
    ap.add_argument("--scans", nargs="+", type=int, default=[1])
    ap.add_argument("--n_stl", type=int, default=3_000_000)
    ap.add_argument("--n_data", type=int, default=8_000_000)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    for i, s in enumerate(a.scans):
        make_scene(a.gt_dir, s, a.n_stl, a.n_data, a.seed + i, a.ply_dir or None)


if __name__ == "__main__":
    main()
