"""Seeded synthetic scans in the Tanks and Temples and BlendedMVS test layouts, for the scan
readers of eval_pipeline (the real data sets are large and licensed separately).

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

    python -m casmvsnet_pl_b200.synth_scenes --kind tanks --root TNT --n_views 150 --image_wh 1920 1080
"""
from __future__ import annotations

import argparse
import os

import numpy as np

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
