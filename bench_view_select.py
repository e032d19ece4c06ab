"""Timing of the COLMAP scene conversion (casmvsnet_pl_b200/colmap.py):

  kernel   casmvs_view_scores_fwd on a Tanks-and-Temples-sized sparse model (synth_scenes.
           sparse_tracks: 300 images, 5e5 points, tracks of 3..11 images, mean 7), inputs already
           on the device, CUDA events around each call (the call includes its one stream
           synchronisation); median of --reps calls after --warmup
  oracle   the vectorised float64 numpy restatement (oracle/view_select_oracle.view_scores_vec)
           on the same model, host wall clock, one call
  scan     one `eval_pipeline --dataset_name colmap` run end to end (model read, view selection,
           depth maps, fusion, PLY) on a synthetic capture (synth_scenes.make_colmap, --scan_views
           views of 1920x1080 / 2400x1350, --img_wh 1152 864, randomly initialised network),
           host wall clock; the first run includes one-time set-up, the second is reported as
           steady state

Prints the card's name and power limit, then one JSON line.  Everything it writes goes to a
temporary directory.

    python bench_view_select.py [--reps 20] [--warmup 3] [--scan_views 16] [--no_scan]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from casmvsnet_pl_b200 import _lib, synth_scenes  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power = (x.strip() for x in out[0].split(","))
        return name, power
    except Exception:                                   # noqa: BLE001
        return torch.cuda.get_device_name(0), "not measured"


def time_kernel(c, xyz, ptr, img, reps, warmup):
    dev = torch.device("cuda:0")
    ct = torch.as_tensor(c, dtype=torch.float64, device=dev)
    pt = torch.as_tensor(xyz, dtype=torch.float64, device=dev)
    pp = torch.as_tensor(ptr, dtype=torch.int64, device=dev)
    it = torch.as_tensor(img, dtype=torch.int32, device=dev)
    n, npts = len(c), len(xyz)
    out = torch.empty(n, n, dtype=torch.float64, device=dev)
    lib = _lib.load()
    nbytes = lib.casmvs_view_scores_workspace_bytes(n, npts, 0)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())        # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call():
        _lib.check(lib.casmvs_view_scores_fwd(vp(ct), vp(pt), vp(pp), vp(it), n, npts, vp(out),
                                              vp(ws), nbytes, st), "view_scores")
    for _ in range(warmup):
        call()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(np.min(ms)), out.cpu().numpy(), nbytes


def time_scan(n_views, img_wh):
    from casmvsnet_pl_b200 import eval_pipeline as ep
    with tempfile.TemporaryDirectory() as d:
        root = os.path.join(d, "capture")
        synth_scenes.make_colmap(root, n_views=n_views, image_wh=(1920, 1080), depth=3.0,
                                 n_points=20000, seed=0)
        argv = ["--dataset_name", "colmap", "--root_dir", root, "--out", os.path.join(d, "out"),
                "--img_wh", str(img_wh[0]), str(img_wh[1])]
        times = []
        for _ in range(2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ep.main(argv)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        with open(os.path.join(d, "out", "capture", "pair.txt")) as f:
            n_refs = int(f.readline())
    return times, n_refs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--scan_views", type=int, default=16)
    ap.add_argument("--no_scan", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_view_select.py needs a GPU"
    name, power = card()
    print(f"card: {name}, power limit {power}")
    c, xyz, ptr, img = synth_scenes.sparse_tracks(300, 500_000, (3, 11), seed=0)
    t = np.diff(ptr)
    n_pairs = int((t * (t - 1) // 2).sum())
    k_med, k_min, got, nbytes = time_kernel(c, xyz, ptr, img, a.reps, a.warmup)
    from oracle import view_select_oracle as O
    t0 = time.perf_counter()
    want = O.view_scores_vec(c, xyz, ptr, img, 300)
    oracle_s = time.perf_counter() - t0
    err = float((np.abs(got - want) / (1 + want)).max())
    res = {"metric": "view_scores", "card": name, "power_limit": power, "n_img": 300,
           "n_pts": len(xyz), "mean_track": float(t.mean()), "n_pairs": n_pairs,
           "workspace_mb": nbytes / 2 ** 20, "kernel_ms_median": k_med, "kernel_ms_min": k_min,
           "pairs_per_s": n_pairs / (k_med / 1e3), "oracle_numpy_s": oracle_s,
           "max_rel_err_vs_oracle": err}
    if a.no_scan:
        res["scan_s"] = "not measured"
    else:
        times, n_refs = time_scan(a.scan_views, (1152, 864))
        res.update({"scan_views": a.scan_views, "scan_ref_views": n_refs, "scan_img_wh": [1152, 864],
                    "scan_first_s": times[0], "scan_s": times[1]})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
