"""Timing of the undistortion of distorted COLMAP views (csrc/undistort.cu, io.undistort_u8):

  kernel   casmvs_undistort_u8_fwd on 150 views of 1920x1080 OPENCV and on 50 views of
           4032x3024 SIMPLE_RADIAL (a phone's 12 MP), inputs already on the device: one launch
           over all views of a set (one map, N images), and the pipeline's shape, one launch per
           view with its two decodes (N = 2).  CUDA events, median of --reps after --warmup.
           Achieved bytes/s = (bytes read + bytes written) / time, each view's image read once and
           its undistorted image written once, over the 3.35 TB/s HBM3 data-sheet bandwidth of
           the H100 SXM
  remap    cv2.remap(INTER_LINEAR, float32 maps) of the same views on the host, for context;
           host wall clock over all views of the set
  scene    eval_pipeline.SceneImages over a capture of 150 JPEG views of 1920x1080 (decode with
           Pillow and cv2, upload, resize to 1152x864), with a PINHOLE camera and with the same
           views as an OPENCV camera (undistorted first); host wall clock to a device synchronise,
           the second of two builds

Prints the card's name and power limit, then one JSON line.  Everything it writes goes to a
temporary directory.

    python bench_undistort.py [--reps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_view_select import card  # noqa: E402
from casmvsnet_pl_b200 import colmap, io, synth_scenes  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SETS = {"opencv_1920x1080": ("OPENCV", 1920, 1080, 150,
                             [1500.0, 1510.0, 957.3, 541.8, -0.11, 0.04, 4e-4, -3e-4]),
        "simple_radial_4032x3024": ("SIMPLE_RADIAL", 4032, 3024, 50, [3200.0, 2015.6, 1512.3, -0.07])}


def _views(n, w, h, distinct=6, seed=0):
    """n host views (n,h,w,3) uint8: `distinct` blurred-noise images repeated."""
    rng = np.random.default_rng(seed)
    base = [synth_scenes._image(rng, w, h) for _ in range(distinct)]
    return np.stack([base[i % distinct] for i in range(n)])


def _events(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def time_set(model, w, h, n, prm, reps, warmup):
    import cv2
    w2, h2, pin = colmap.undistorted_camera(1, model, w, h, prm)
    src, dst = (colmap.MODEL_IDS[model][0], w, h, prm), (w2, h2, pin)
    host = _views(n, w, h)
    dev = torch.from_numpy(host).cuda()
    out = torch.empty(n, h2, w2, 3, dtype=torch.uint8, device="cuda")
    nbytes = n * (h * w + h2 * w2) * 3
    one_ms = _events(lambda: io.undistort_u8(dev, src, dst, out=out), reps, warmup)

    def pairs():
        for i in range(0, n - 1, 2):
            io.undistort_u8(dev[i:i + 2], src, dst, out=out[i:i + 2])
    pair_ms = _events(pairs, max(3, reps // 4), 1)
    # the host route: the same map as float32 maps for cv2.remap (BORDER_CONSTANT 0)
    from oracle import undistort_oracle as O
    sx, sy, _ = O.source_map(model, prm, pin, (w2, h2), (w, h))
    mx, my = sx.astype(np.float32), sy.astype(np.float32)
    cv2.remap(host[0], mx, my, cv2.INTER_LINEAR)
    t0 = time.perf_counter()
    for i in range(n):
        cv2.remap(host[i], mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT)
    remap_s = time.perf_counter() - t0
    same = bool(np.array_equal(out[0].cpu().numpy(), O.remap(host[:1], model, prm, pin, (w2, h2))[0]))
    return {"model": model, "views": n, "src_wh": [w, h], "dst_wh": [w2, h2],
            "bytes_per_launch": nbytes, "kernel_ms_one_launch": one_ms,
            "kernel_tb_per_s": nbytes / (one_ms / 1e3) / 1e12,
            "kernel_share_of_hbm": nbytes / (one_ms / 1e3) / HBM_BYTES_PER_S,
            "kernel_ms_pairs": pair_ms, "pairs_tb_per_s": nbytes / (pair_ms / 1e3) / 1e12,
            "cv2_remap_host_s": remap_s, "equals_oracle_view0": same}


def time_scene(n, reps=2):
    from PIL import Image

    from casmvsnet_pl_b200.eval_pipeline import SceneImages
    model, w, h, _, prm = SETS["opencv_1920x1080"]
    w2, h2, pin = colmap.undistorted_camera(1, model, w, h, prm)
    cams = {v: ((colmap.MODEL_IDS[model][0], w, h, prm), (w2, h2, pin)) for v in range(n)}
    res = {}
    with tempfile.TemporaryDirectory() as d:
        views = _views(6, w, h, seed=1)
        for i in range(6):
            Image.fromarray(views[i]).save(os.path.join(d, f"v{i}.jpg"), quality=92)
        paths = {v: os.path.join(d, f"v{v % 6}.jpg") for v in range(n)}
        for tag, cameras in (("pinhole", None), ("opencv", cams)):
            for _ in range(reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                imgs = SceneImages(paths, (1152, 864), "cuda:0", cameras=cameras)
                torch.cuda.synchronize()
                res[f"scene_{tag}_s"] = time.perf_counter() - t0
                del imgs
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_undistort.py needs a GPU"
    name, power = card()
    print(f"card: {name}, power limit {power}")
    res = {"metric": "undistort", "card": name, "power_limit": power}
    for tag, (model, w, h, n, prm) in SETS.items():
        res[tag] = time_set(model, w, h, n, prm, a.reps, a.warmup)
        torch.cuda.empty_cache()
    res.update(time_scene(150))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
