"""DTU point-cloud scoring on the GPU: accuracy, completeness and overall of a fused cloud against
the DTU ground truth, restating the reference's MATLAB scorer (paths relative to the reference
root):

    thinning to 0.2 mm          evaluations/dtu/reducePts_haa.m, PointCompareMain.m:7
    Ddata / Dstl (60 mm cap)    MaxDistCP.m, PointCompareMain.m:20-28
    DataInMask                  PointCompareMain.m:32-41
    StlAbovePlane               PointCompareMain.m:53
    statistics                  BaseEvalMain_web.m:59-68, ComputeStat_web.m:49-65,76-78

Ground truth as the MATLAB reads it:

    <gt>/Points/stl/stl{NNN}_total.ply
    <gt>/ObsMask/ObsMask{N}_10.mat      ObsMask, BB, Res
    <gt>/ObsMask/Plane{N}.mat           P

Thinning and the nearest-neighbour searches run in csrc/pcd_eval.cu; the cell-key sort and
run-length scan that build their grids, the masks and the statistics are torch ops on the device.
The MATLAB visits points in an unseeded random order, so its scores vary from run to run; here the
order is torch.randperm on the CPU seeded by `seed`, and the same seed and input order give the
same kept set on every run and every GPU.

    python -m casmvsnet_pl_b200.dtu_eval --ply_dir results/dtu/points --gt_dir DTU_GT [--scans 1 4]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import time

import numpy as np
import torch

from . import _lib, io, ops

USED_SETS = (1, 4, 9, 10, 11, 12, 13, 15, 23, 24, 29, 32, 33, 34, 48, 49, 62, 75, 77, 110, 114, 118)
DST = 0.2            # BaseEvalMain_web.m:25
MAX_DIST = 60.0      # PointCompareMain.m:20
OUTLIER = 20.0       # BaseEvalMain_web.m:59, ComputeStat_web.m
MARGIN = 10          # PointCompareMain.m:17
_OUTSIDE = torch.iinfo(torch.int64).max
NN_CELL = 1.0        # mm: fine cell edge of the nearest-neighbour grid (super cells of 8 mm)


# ------------------------------------------------------------------------------ ground truth
def _loadmat(path):
    import scipy.io                    # optional dependency, only needed to score
    if not os.path.isfile(path):
        raise FileNotFoundError(path)
    return scipy.io.loadmat(path)


def load_obs_mask(gt_dir, scan):
    """ObsMask{N}_10.mat -> (ObsMask bool (X,Y,Z) in stored axis order, BB (2,3) float64, Res)."""
    m = _loadmat(os.path.join(gt_dir, "ObsMask", f"ObsMask{scan}_{MARGIN}.mat"))
    bb = np.asarray(m["BB"], dtype=np.float64).reshape(2, 3)
    return np.asarray(m["ObsMask"]).astype(bool), bb, float(np.asarray(m["Res"]).reshape(-1)[0])


def load_plane(gt_dir, scan):
    """Plane{N}.mat -> P (4,) float64 (StlAbovePlane: P . [q; 1] > 0)."""
    return np.asarray(_loadmat(os.path.join(gt_dir, "ObsMask", f"Plane{scan}.mat"))["P"],
                      dtype=np.float64).reshape(4)


def read_points(path):
    """x, y, z of a PLY's vertices -> (N,3) float32 ndarray."""
    v = io.read_ply(path)
    return np.ascontiguousarray(np.stack([v["x"], v["y"], v["z"]], axis=1), dtype=np.float32)


def stl_path(gt_dir, scan):
    return os.path.join(gt_dir, "Points", "stl", f"stl{scan:03d}_total.ply")


def block_grid(bb, max_dist=MAX_DIST):
    """The query region of MaxDistCP.m:5-18 -> (lo, hi): q is scored iff lo <= q < hi on every
    axis.  hi is computed as the MATLAB computes the last block's upper face,
    (BB1 + floor((BB2 - BB1)/max_dist) * max_dist) + max_dist, in double."""
    bb = np.asarray(bb, dtype=np.float64).reshape(2, 3)
    rng = np.floor((bb[1] - bb[0]) / max_dist)
    return bb[0].copy(), (bb[0] + rng * max_dist) + max_dist


# ------------------------------------------------------------------------------ device steps
def _check_points(name, points):
    if not (torch.is_tensor(points) and points.is_cuda and points.dtype == torch.float32
            and points.dim() == 2 and points.shape[1] == 3):
        raise ValueError(f"{name} must be a float32 CUDA tensor of shape (N,3)")
    return points.contiguous()


def visiting_rank(n, seed):
    """rank[i] = position of point i in the visiting order torch.randperm(n) seeded by `seed`."""
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(int(seed)))
    rank = torch.empty(n, dtype=torch.int32)
    rank[perm] = torch.arange(n, dtype=torch.int32)
    return rank


def _cells(keys_sorted):
    ukeys, counts = torch.unique_consecutive(keys_sorted, return_counts=True)
    start = torch.zeros(len(ukeys) + 1, device=keys_sorted.device, dtype=torch.int32)
    torch.cumsum(counts, 0, out=start[1:])
    return ukeys, start


def thin(points, dst=DST, seed=0, timings=None):
    """Indices (ascending int64, on the device) of the points reducePts_haa.m keeps for the visiting
    order visiting_rank(N, seed): the lexicographically-first maximal subset pairwise more than
    `dst` apart."""
    pts = _check_points("points", points)
    if not dst > 0:
        raise ValueError("dst must be > 0")
    n = pts.shape[0]
    if n == 0:
        return torch.zeros(0, device=pts.device, dtype=torch.int64)
    if not bool(torch.isfinite(pts).all()):
        raise ValueError("points must be finite")
    t0 = _sync_time()
    lo = pts.min(0).values.double().cpu().numpy()
    ext = float((pts.max(0).values.double().cpu().numpy() - lo).max())
    cell = max(dst * (1 + 1e-6), ext / ((1 << 20) - 4))     # > dst: neighbours are 1 cell away
    dims = [int(math.floor(ext / cell)) + 2] * 3
    keys = ops.pcd_cell_keys(pts, lo, cell, dims, sub=1)
    keys, order = torch.sort(keys, stable=True)
    pts_s = pts[order].contiguous()
    rank = visiting_rank(n, seed).to(pts.device)[order].contiguous()
    ukeys, start = _cells(keys)
    ws = ops.pcd_thin_prepare(ukeys, start, n, dims)
    t1 = _sync_time()
    state = torch.zeros(n, device=pts.device, dtype=torch.uint8)
    undecided = torch.zeros(1, device=pts.device, dtype=torch.int32)
    rounds = 0
    while True:
        ops.pcd_thin_round(pts_s, rank, start, dst, state, undecided, ws)
        rounds += 1
        if int(undecided.item()) == 0:
            break
    kept = torch.sort(order[state == 1]).values
    t2 = _sync_time()
    if timings is not None:
        timings["thin_grid_s"] = t1 - t0
        timings["thin_rounds_s"] = t2 - t1
        timings["thin_rounds"] = rounds
    return kept


def capped_nn(queries, targets, box_lo, box_hi, cap=MAX_DIST, cell=NN_CELL, timings=None, tag="nn"):
    """MaxDistCP.m: min(nearest-target distance, cap) (float64, device) for queries with
    box_lo <= q < box_hi on every axis, cap for the others."""
    q = _check_points("queries", queries)
    t = _check_points("targets", targets)
    box_lo = np.asarray(box_lo, dtype=np.float64).reshape(3)
    box_hi = np.asarray(box_hi, dtype=np.float64).reshape(3)
    t0 = _sync_time()
    # targets farther than the cap from every scored query cannot change a distance
    org = box_lo - cap
    ext = float(((box_hi + cap) - org).max())
    h = max(float(cell), ext / (8 * 255))                    # at most 256^3 super cells
    sdims = [int(math.floor(e / (8 * h))) + 2 for e in ((box_hi + cap) - org)]
    keys = ops.pcd_cell_keys(t, org, h, [8 * s for s in sdims], sub=8)
    keys, order = torch.sort(keys)
    m = int(torch.searchsorted(keys, torch.tensor([_OUTSIDE], device=keys.device)).item())
    keys, tgt = keys[:m], t[order[:m]].contiguous()
    ukeys, start = _cells(keys)
    nsuper = sdims[0] * sdims[1] * sdims[2]
    super_begin = torch.searchsorted(ukeys >> 9, torch.arange(nsuper + 1, device=q.device)).int()
    t1 = _sync_time()
    dist = ops.pcd_capped_nn(q, tgt, ukeys, start, super_begin, org, h, sdims, box_lo, box_hi, cap)
    t2 = _sync_time()
    if timings is not None:
        timings[f"{tag}_grid_s"] = t1 - t0
        timings[f"{tag}_search_s"] = t2 - t1
    return dist


def round_half_away(x):
    """MATLAB round(): halves away from zero (torch.round rounds them to even)."""
    t = torch.trunc(x)
    return t + torch.sign(x) * ((x - t).abs() >= 0.5).to(x.dtype)


def data_in_mask(points, obs_mask, bb, res):
    """PointCompareMain.m:32-41: v = round((q - BB1)/Res + 1) in double, inside iff
    1 <= v <= size(ObsMask) on every axis and ObsMask(v)."""
    pts = _check_points("points", points)
    mask = obs_mask if torch.is_tensor(obs_mask) else torch.from_numpy(np.ascontiguousarray(obs_mask))
    mask = mask.to(pts.device, torch.bool)
    b1 = torch.as_tensor(np.asarray(bb, dtype=np.float64).reshape(2, 3)[0], device=pts.device)
    v = round_half_away((pts.double() - b1) / float(res) + 1)
    size = torch.tensor(mask.shape, device=pts.device, dtype=torch.float64)
    inside = ((v >= 1) & (v <= size)).all(1)
    out = torch.zeros(pts.shape[0], device=pts.device, dtype=torch.bool)
    idx = (v[inside] - 1).long()
    out[inside] = mask[idx[:, 0], idx[:, 1], idx[:, 2]]
    return out


def stl_above_plane(points, plane):
    """PointCompareMain.m:53: ((P1*x + P2*y) + P3*z) + P4 > 0 in double."""
    pts = _check_points("points", points).double()
    P = [float(v) for v in np.asarray(plane, dtype=np.float64).reshape(4)]
    return ((P[0] * pts[:, 0] + P[1] * pts[:, 1]) + P[2] * pts[:, 2]) + P[3] > 0


def matlab_stats(d, sel, max_dist=OUTLIER):
    """Mean, median (mean of the two middle values for an even count), unbiased variance and count
    of d[sel & d < max_dist], as ComputeStat_web.m takes them (NaN for an empty set, var 0 for
    one value)."""
    x = d[sel & (d < max_dist)].double()
    n = int(x.numel())
    if n == 0:
        return dict(mean=math.nan, median=math.nan, var=math.nan, n=0)
    xs = torch.sort(x).values
    med = xs[n // 2] if n % 2 else (xs[n // 2 - 1] + xs[n // 2]) / 2
    var = float(x.var(correction=1).item()) if n > 1 else 0.0
    return dict(mean=float(x.mean().item()), median=float(med.item()), var=var, n=n)


def _sync_time():
    torch.cuda.synchronize()
    return time.perf_counter()


# ------------------------------------------------------------------------------ one scan
def evaluate_scan(points, scan, gt_dir, dst=DST, seed=0, device="cuda:0", return_arrays=False):
    """Scores one DTU scan.  `points` is a float32 CUDA (N,3) tensor (such as fusion.fuse_scan's
    output) or the path of a PLY; `scan` the DTU scan number.  Returns a dict with acc, comp,
    overall (mm), the medians, variances and counts of both sides, point counts and
    device-synchronised timings per phase (time_s).  return_arrays adds the device tensors kept
    (thinned indices), Ddata, Dstl, data_in_mask and stl_above_plane."""
    if isinstance(scan, bool) or not isinstance(scan, (int, np.integer)) or scan < 0:
        raise ValueError(f"scan must be a DTU scan number, got {scan!r}")
    if not dst > 0:
        raise ValueError("dst must be > 0")
    if not os.path.isdir(gt_dir):
        raise FileNotFoundError(gt_dir)
    if isinstance(points, (str, os.PathLike)):
        src = None
    elif torch.is_tensor(points):
        _check_points("points", points)
        src = points
    else:
        raise TypeError("points must be a CUDA (N,3) tensor or a PLY path")
    times = {}
    t0 = time.perf_counter()
    if src is None:
        dev = torch.device(device)
        _require_device(dev)
        with torch.cuda.device(dev):
            src = torch.from_numpy(read_points(points)).to(dev)
    with torch.cuda.device(src.device):
        stl = torch.from_numpy(read_points(stl_path(gt_dir, scan))).to(src.device)
        obs, bb, res = load_obs_mask(gt_dir, scan)
        plane = load_plane(gt_dir, scan)
        lo, hi = block_grid(bb)
        t1 = _sync_time()
        times["load_s"] = t1 - t0
        kept = thin(src, dst, seed, timings=times)
        data = src[kept].contiguous()
        t2 = _sync_time()
        times["thin_s"] = t2 - t1
        d_data = capped_nn(data, stl, lo, hi, timings=times, tag="ddata")
        t3 = _sync_time()
        times["ddata_s"] = t3 - t2
        d_stl = capped_nn(stl, data, lo, hi, timings=times, tag="dstl")
        t4 = _sync_time()
        times["dstl_s"] = t4 - t3
        in_mask = data_in_mask(data, obs, bb, res)
        above = stl_above_plane(stl, plane)
        acc = matlab_stats(d_data, in_mask)
        comp = matlab_stats(d_stl, above)
        times["stats_s"] = _sync_time() - t4
    times["total_s"] = time.perf_counter() - t0
    out = dict(scan=int(scan), acc=acc["mean"], comp=comp["mean"],
               overall=(acc["mean"] + comp["mean"]) / 2,
               acc_median=acc["median"], comp_median=comp["median"],
               acc_var=acc["var"], comp_var=comp["var"], n_acc=acc["n"], n_comp=comp["n"],
               n_data=int(src.shape[0]), n_thinned=int(data.shape[0]), n_stl=int(stl.shape[0]),
               dst=float(dst), seed=int(seed), time_s=times)
    if return_arrays:
        out.update(kept=kept, Ddata=d_data, Dstl=d_stl, data_in_mask=in_mask, stl_above_plane=above)
    return out


def _require_device(dev):
    if dev.type != "cuda" or not torch.cuda.is_available():
        raise _lib.CasMVSError("DTU scoring runs on the GPU (no CPU fallback)")


def summarize(results):
    """Multi-scan summary (ComputeStat_web.m:76-78): mean of the per-scan means."""
    results = list(results)
    if not results:
        raise ValueError("summarize needs at least one scan result")
    acc = float(np.mean([r["acc"] for r in results]))
    comp = float(np.mean([r["comp"] for r in results]))
    return dict(acc=acc, comp=comp, overall=(acc + comp) / 2, n_scans=len(results),
                scans=[int(r["scan"]) for r in results])


def scan_number(name):
    """'scan9' / 'scan9.ply' / 9 -> 9."""
    import re
    if isinstance(name, (int, np.integer)):
        return int(name)
    m = re.fullmatch(r"(?:scan)?(\d+)(?:\.ply)?", os.path.basename(str(name)))
    if not m:
        raise ValueError(f"not a DTU scan name: {name!r}")
    return int(m.group(1))


def _fmt(r):
    t = r["time_s"]
    return (f"scan{r['scan']}: acc {r['acc']:.4f}  comp {r['comp']:.4f}  overall {r['overall']:.4f} mm"
            f"  ({r['n_data']} -> {r['n_thinned']} points, {r['n_stl']} STL)  time: "
            + " ".join(f"{k[:-2]} {v:.3f}s" for k, v in t.items() if k.endswith("_s")))


def main(argv=None):
    ap = argparse.ArgumentParser(description="Score fused DTU point clouds (scan{N}.ply) on the GPU.")
    ap.add_argument("--ply_dir", required=True)
    ap.add_argument("--gt_dir", required=True)
    ap.add_argument("--scans", nargs="+", type=int, default=list(USED_SETS))
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--dst", type=float, default=DST)
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--out", default="")
    a = ap.parse_args(argv)
    results = []
    for s in a.scans:
        r = evaluate_scan(os.path.join(a.ply_dir, f"scan{s}.ply"), s, a.gt_dir, a.dst, a.seed, a.device)
        print(_fmt(r), flush=True)
        results.append(r)
    summ = summarize(results)
    print(f"mean over {summ['n_scans']} scans: acc {summ['acc']:.4f}  comp {summ['comp']:.4f}  "
          f"overall {summ['overall']:.4f} mm")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(scans=results, summary=summ), f, indent=1)
    return summ


if __name__ == "__main__":
    main()
