"""Tanks and Temples training-set scoring on the GPU: align a reconstruction to the ground truth,
refine the alignment with three ICP stages, then precision, recall and F-score at the scene's tau.

This is the protocol of the Tanks and Temples toolbox (run.py, registration.py, evaluation.py),
stated here as this project's rules; neither the toolbox nor Open3D is needed, and agreement with
them has not been checked.

Ground truth, in <gt>/<Scene>/:

    <Scene>.ply              the laser scan
    <Scene>.json             Open3D SelectionPolygonVolume (orthogonal_axis, axis_min, axis_max,
                             bounding_polygon)
    <Scene>_trans.txt        4x4 from the official COLMAP SfM frame to the ground-truth frame
    <Scene>_COLMAP_SfM.log   the official SfM camera poses

1. Alignment (host, float64): the reconstruction's camera centres are paired with the SfM centres
   mapped by _trans.txt (by order, or by image name with `images`), and a seeded RANSAC of
   Umeyama similarities (100 000 hypotheses of 6 distinct pairs, inlier residual < 0.2; best =
   most inliers, then lower inlier RMSE, then drawn first) gives T0, refitted on the inliers.
2. Three ICP refinements (GPU): transform the reconstruction by the stage's initial T (double,
   rounded to float32), crop both clouds, downsample both (voxel tau with d = 80 tau, voxel tau/2
   with d = 20 tau, uniform with d = 2 tau), then point-to-point ICP with scale from the identity
   (at most 20 iterations; stop when fitness and RMSE both move less than 1e-6).
3. Scores (GPU): both clouds cropped and downsampled to voxel tau/2; d1 = reconstruction ->
   ground truth, d2 = ground truth -> reconstruction nearest distances (capped at 5 tau);
   precision = #(d1 < tau)/|d1|, recall = #(d2 < tau)/|d2|, F = 2PR/(P+R), and the cumulative
   curves over the edges k tau/100, k < 500.

Crop, voxel means and nearest neighbours are csrc/tnt_eval.cu and csrc/pcd_eval.cu; the key sorts,
run-length scans and histograms are torch ops on the device.  Same inputs and seed give the same
scores and transforms, bit for bit.

    python -m casmvsnet_pl_b200.tnt_eval --ply points/Barn.ply --run_dir results/colmap/Barn \\
        --gt_dir TNT_GT --scene Barn [--images Barn/images] [--out scores.json]
    python -m casmvsnet_pl_b200.tnt_eval --mesh mesh/Barn.ply --run_dir results/colmap/Barn ...

A mesh is scored through its surface samples at tau / 4 (mesh_sample.py); alignment uses only
the cameras, so it is the same as for a cloud.
"""
from __future__ import annotations

import argparse
import glob
import json
import math
import os
import time

import numpy as np
import torch

from . import _lib, io, ops

TAU = {"Barn": 0.01, "Caterpillar": 0.005, "Church": 0.025, "Courthouse": 0.025,
       "Ignatius": 0.003, "Meetinghouse": 0.01, "Truck": 0.005}
RANSAC_HYPOTHESES = 100_000
RANSAC_SAMPLE = 6
RANSAC_INLIER = 0.2
ICP_MAX_ITER = 20
ICP_CONVERGE = 1e-6
UNIFORM_MAX = 4_000_000
N_EDGES = 500
MAX_GRID = 1 << 20
_OUTSIDE = torch.iinfo(torch.int64).max


# ------------------------------------------------------------------------------ readers
def _numbers(path, text, count, what):
    try:
        vals = [float(x) for x in text.split()]
    except ValueError:
        raise ValueError(f"{path}: {what} holds a token that is not a number") from None
    if len(vals) != count or not all(math.isfinite(v) for v in vals):
        raise ValueError(f"{path}: {what} must be {count} finite numbers, got {len(vals)}")
    return vals


def read_trans(path):
    """<Scene>_trans.txt -> (4,4) float64."""
    with open(path) as f:
        T = np.array(_numbers(path, f.read(), 16, "the transform"), np.float64).reshape(4, 4)
    if not np.array_equal(T[3], [0, 0, 0, 1]) or abs(np.linalg.det(T[:3, :3])) < 1e-300:
        raise ValueError(f"{path}: the transform's last row must be 0 0 0 1 and its 3x3 invertible")
    return T


def read_log(path):
    """A trajectory .log -> (n,4,4) float64 camera-to-world matrices: each entry is a line of
    three integers and four lines of the matrix."""
    with open(path) as f:
        lines = [ln for ln in f.read().splitlines() if ln.strip()]
    if len(lines) % 5:
        raise ValueError(f"{path}: a .log entry is 5 lines (3 integers, then 4x4); "
                         f"{len(lines)} lines")
    poses = []
    for k in range(0, len(lines), 5):
        head = lines[k].split()
        if len(head) != 3 or not all(h.lstrip("-").isdigit() for h in head):
            raise ValueError(f"{path}: entry {k // 5} must start with a line of 3 integers")
        M = np.array(_numbers(path, " ".join(lines[k + 1:k + 5]), 16, f"entry {k // 5}'s matrix"),
                     np.float64).reshape(4, 4)
        poses.append(M)
    return np.stack(poses) if poses else np.zeros((0, 4, 4))


def read_crop(path):
    """Open3D SelectionPolygonVolume JSON -> (axis 0/1/2, axis_min, axis_max, polygon (m,2) of
    the (u, v) plane coordinates: (y, z), (x, z) or (x, y) for axis X, Y or Z)."""
    try:
        with open(path) as f:
            data = json.load(f)
    except json.JSONDecodeError as e:
        raise ValueError(f"{path}: not a JSON file ({e})") from None
    if not isinstance(data, dict):
        raise ValueError(f"{path}: a crop file holds one JSON object")
    ax = data.get("orthogonal_axis")
    if not isinstance(ax, str) or ax.upper() not in ("X", "Y", "Z"):
        raise ValueError(f"{path}: orthogonal_axis must be X, Y or Z")
    axis = "XYZ".index(ax.upper())
    lim = []
    for key in ("axis_min", "axis_max"):
        v = data.get(key)
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
            raise ValueError(f"{path}: {key} must be a finite number")
        lim.append(float(v))
    if not lim[0] <= lim[1]:
        raise ValueError(f"{path}: axis_min must be <= axis_max")
    poly = data.get("bounding_polygon")
    if not isinstance(poly, list) or len(poly) < 3:
        raise ValueError(f"{path}: bounding_polygon must be a list of at least 3 points")
    pts = []
    for p in poly:
        if not (isinstance(p, list) and len(p) == 3 and all(
                isinstance(x, (int, float)) and not isinstance(x, bool) and math.isfinite(x) for x in p)):
            raise ValueError(f"{path}: bounding_polygon entries must be 3 finite numbers")
        pts.append(p)
    u, v = plane_axes(axis)
    P = np.array(pts, np.float64)
    return axis, lim[0], lim[1], np.ascontiguousarray(P[:, [u, v]])


def plane_axes(axis):
    return {0: (1, 2), 1: (0, 2), 2: (0, 1)}[axis]


def read_points(path):
    v = io.read_ply(path)
    return np.ascontiguousarray(np.stack([v["x"], v["y"], v["z"]], axis=1), dtype=np.float32)


def gt_paths(gt_dir, scene):
    d = os.path.join(gt_dir, scene)
    return dict(ply=os.path.join(d, f"{scene}.ply"), crop=os.path.join(d, f"{scene}.json"),
                trans=os.path.join(d, f"{scene}_trans.txt"),
                log=os.path.join(d, f"{scene}_COLMAP_SfM.log"))


def scene_tau(scene, tau=None):
    if tau is not None:
        if not tau > 0:
            raise ValueError("tau must be > 0")
        return float(tau)
    if scene not in TAU:
        raise ValueError(f"no tau for scene {scene!r}: the training scenes are {sorted(TAU)}; "
                         "give --tau for any other scene")
    return TAU[scene]


# ------------------------------------------------------------------------------ trajectories
class Trajectory:
    """Camera centres (n,3) float64 and, when known, each camera's image name."""

    def __init__(self, centres, names=None):
        self.centres = np.asarray(centres, np.float64).reshape(-1, 3)
        self.names = list(names) if names is not None else None

    def __len__(self):
        return len(self.centres)


def trajectory_from_log(path):
    P = read_log(path)
    return Trajectory(P[:, :3, 3])


def trajectory_from_run(run_dir):
    """The cameras a run recorded: <run_dir>/cams/{vid:08d}_cam.txt (world -> camera extrinsic)
    and view_names.txt (view id -> image name), in view order."""
    cams = sorted(glob.glob(os.path.join(run_dir, "cams", "*_cam.txt")))
    if not cams:
        raise FileNotFoundError(f"{run_dir}: no cams/*_cam.txt")
    names = {}
    vn = os.path.join(run_dir, "view_names.txt")
    if os.path.isfile(vn):
        with open(vn) as f:
            for ln in f:
                if ln.strip():
                    vid, name = ln.strip().split(maxsplit=1)
                    names[int(vid)] = name
    centres, nm = [], []
    for p in cams:
        vid = int(os.path.basename(p).split("_")[0])
        with open(p) as f:
            lines = f.read().splitlines()
        E = np.array(_numbers(p, " ".join(lines[1:5]), 16, "the extrinsic"), np.float64).reshape(4, 4)
        centres.append(-E[:3, :3].T @ E[:3, 3])
        nm.append(names.get(vid))
    return Trajectory(np.array(centres), nm if names else None)


def pair_cameras(recon, gt_count, images=None):
    """(recon indices, gt frame indices) of the camera pairs.  Without `images`, by order (the
    counts must agree); with it, a camera pairs with frame k when its image name is the k-th name
    of the directory's sorted listing."""
    if images is None:
        if len(recon) != gt_count:
            raise ValueError(f"the reconstruction has {len(recon)} cameras and the ground-truth "
                             f"log {gt_count}: pair them by image name with --images DIR")
        return np.arange(len(recon)), np.arange(gt_count)
    if recon.names is None or any(n is None for n in recon.names):
        raise ValueError("pairing by --images needs each camera's image name (view_names.txt)")
    listing = sorted(f for f in os.listdir(images) if not f.startswith("."))
    if len(listing) != gt_count:
        raise ValueError(f"{images} lists {len(listing)} images and the ground-truth log has "
                         f"{gt_count} frames")
    pos = {name: k for k, name in enumerate(listing)}
    ri, gi = [], []
    for i, name in enumerate(recon.names):
        k = pos.get(os.path.basename(name))
        if k is None:
            raise ValueError(f"image {name!r} of the reconstruction is not in {images}")
        ri.append(i)
        gi.append(k)
    return np.array(ri, np.int64), np.array(gi, np.int64)


# ------------------------------------------------------------------------------ alignment
def _apply(T, p):
    return p @ T[:3, :3].T + T[:3, 3]


def umeyama_from_stats(n, ms, mt, var, sigma):
    """Umeyama with scale from means ms, mt, var = mean|s - ms|^2 and sigma = mean (t - mt)(s -
    ms)^T -> 4x4 (t ~ c R s + t0)."""
    U, D, Vt = np.linalg.svd(sigma)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1
    R = U @ np.diag(S) @ Vt
    c = (D * S).sum() / var
    T = np.eye(4)
    T[:3, :3] = c * R
    T[:3, 3] = mt - c * R @ ms
    return T


def umeyama(src, dst):
    s, d = np.asarray(src, np.float64), np.asarray(dst, np.float64)
    ms, md = s.mean(0), d.mean(0)
    sc, dc = s - ms, d - md
    return umeyama_from_stats(len(s), ms, md, (sc * sc).sum(1).mean(), dc.T @ sc / len(s))


def _umeyama_batch(S, D):
    """Umeyama of each (k,3) pair of S, D (m,k,3) -> (m,4,4); degenerate samples give non-finite
    transforms, which score no inliers."""
    ms, md = S.mean(1), D.mean(1)
    sc, dc = S - ms[:, None], D - md[:, None]
    var = (sc * sc).sum(2).mean(1)
    sigma = np.einsum("mki,mkj->mij", dc, sc) / S.shape[1]
    U, Dg, Vt = np.linalg.svd(sigma)
    sgn = np.where(np.linalg.det(U) * np.linalg.det(Vt) < 0, -1.0, 1.0)
    Sd = np.ones((len(S), 3))
    Sd[:, 2] = sgn
    R = U @ (Sd[:, :, None] * Vt)
    with np.errstate(divide="ignore", invalid="ignore"):
        c = (Dg * Sd).sum(1) / var
    T = np.tile(np.eye(4), (len(S), 1, 1))
    T[:, :3, :3] = c[:, None, None] * R
    T[:, :3, 3] = md - np.einsum("mij,mj->mi", T[:, :3, :3], ms)
    return T


def ransac_align(src, dst, seed=0, n_hyp=RANSAC_HYPOTHESES, sample=RANSAC_SAMPLE,
                 thresh=RANSAC_INLIER, chunk=4096):
    """Seeded RANSAC of similarities dst ~ T src -> (T0 refitted on the inliers, inlier mask)."""
    src, dst = np.asarray(src, np.float64), np.asarray(dst, np.float64)
    n = len(src)
    if n < sample:
        raise ValueError(f"alignment needs at least {sample} camera pairs, got {n}")
    rng = np.random.default_rng(seed)
    best = (-1, math.inf)
    best_T = None
    for c0 in range(0, n_hyp, chunk):
        m = min(chunk, n_hyp - c0)
        pick = np.argsort(rng.random((m, n)), axis=1, kind="stable")[:, :sample]
        T = _umeyama_batch(src[pick], dst[pick])
        with np.errstate(invalid="ignore", over="ignore"):
            pred = np.einsum("mij,nj->mni", T[:, :3, :3], src) + T[:, None, :3, 3]
            res = np.sqrt(((pred - dst[None]) ** 2).sum(2))
            inl = res < thresh
            cnt = inl.sum(1)
            rmse = np.sqrt(np.where(inl, res * res, 0.0).sum(1) / np.maximum(cnt, 1))
        for k in np.lexsort((np.arange(m), rmse, -cnt))[:1]:
            if cnt[k] > best[0] or (cnt[k] == best[0] and rmse[k] < best[1]):
                best, best_T = (int(cnt[k]), float(rmse[k])), T[k]
    if best[0] < 3:
        raise ValueError("alignment found no similarity with 3 or more inlier cameras")
    inl = np.sqrt(((_apply(best_T, src) - dst) ** 2).sum(1)) < thresh
    return umeyama(src[inl], dst[inl]), inl


def align(recon, gt_log_centres, trans, images=None, seed=0):
    ri, gi = pair_cameras(recon, len(gt_log_centres), images)
    if len(ri) < RANSAC_SAMPLE:
        raise ValueError(f"alignment needs at least {RANSAC_SAMPLE} camera pairs, got {len(ri)}")
    dst = _apply(trans, np.asarray(gt_log_centres, np.float64)[gi])
    T0, inl = ransac_align(recon.centres[ri], dst, seed)
    return T0, dict(pairs=int(len(ri)), inliers=int(inl.sum()))


# ------------------------------------------------------------------------------ device steps
def _sync_time():
    torch.cuda.synchronize()
    return time.perf_counter()


class CropVolume:
    def __init__(self, axis, amin, amax, polygon, device):
        self.axis, self.amin, self.amax = int(axis), float(amin), float(amax)
        self.polygon = np.asarray(polygon, np.float64)
        self.poly_dev = torch.from_numpy(self.polygon).to(device)
        u, v = plane_axes(self.axis)
        lo, hi = np.zeros(3), np.zeros(3)
        lo[self.axis], hi[self.axis] = self.amin, self.amax
        lo[[u, v]], hi[[u, v]] = self.polygon.min(0), self.polygon.max(0)
        self.lo, self.hi = lo, hi
        self.centre = (lo + hi) / 2           # the fixed origin of the ICP moments

    def args(self):
        return self.axis, self.amin, self.amax, self.poly_dev


def crop(points, vol, T=None):
    """float32(T p) of the points inside the crop volume, in input order."""
    return ops.tnt_transform_crop(points, T, vol.args())[0]


def _cells(keys_sorted):
    ukeys, counts = torch.unique_consecutive(keys_sorted, return_counts=True)
    start = torch.zeros(len(ukeys) + 1, device=keys_sorted.device, dtype=torch.int32)
    torch.cumsum(counts, 0, out=start[1:])
    return ukeys, start


def voxel_downsample(points, voxel):
    """One float32 point per occupied voxel of edge `voxel` from the cloud's minimum bound minus
    half a voxel, in ascending key order: the mean of its points, summed in double in input
    order."""
    if points.shape[0] == 0:
        return points
    lo = points.min(0).values.double().cpu().numpy()
    hi = points.max(0).values.double().cpu().numpy()
    origin = lo - voxel * 0.5
    dims = [int(v) for v in np.floor((hi - origin) / voxel) + 1]
    if max(dims) >= MAX_GRID:
        raise ValueError(f"voxel {voxel:g} makes a grid of {dims} cells; at most 2^20 - 1 per axis")
    keys = ops.pcd_cell_keys(points, origin, voxel, dims, sub=1)
    keys, order = torch.sort(keys, stable=True)
    _, start = _cells(keys)
    return ops.tnt_voxel_mean(points, order, start)


def uniform_downsample(points, max_points=UNIFORM_MAX):
    n = points.shape[0]
    if n <= max_points:
        return points
    return points[::int(round(n / max_points))].contiguous()


class NNGrid:
    """The capped nearest-neighbour grid (pcd_eval.cu) over `targets` for queries anywhere within
    `cap` of the crop box [lo, hi]."""

    def __init__(self, targets, lo, hi, cap, cell):
        self.cap = float(cap)
        self.targets_all = targets
        self.box_lo = np.asarray(lo, np.float64) - cap
        self.box_hi = np.asarray(hi, np.float64) + cap
        org = self.box_lo - cap
        span = (self.box_hi + cap) - org
        self.h = max(float(cell), float(span.max()) / (8 * 255))
        self.sdims = [int(math.floor(e / (8 * self.h))) + 2 for e in span]
        self.org = org
        keys = ops.pcd_cell_keys(targets, org, self.h, [8 * s for s in self.sdims], sub=8)
        keys, order = torch.sort(keys, stable=True)
        m = int(torch.searchsorted(keys, torch.tensor([_OUTSIDE], device=keys.device)).item())
        self.index = order[:m].contiguous()
        self.tgt = targets[self.index].contiguous()
        self.ukeys, self.start = _cells(keys[:m])
        nsuper = self.sdims[0] * self.sdims[1] * self.sdims[2]
        self.super_begin = torch.searchsorted(self.ukeys >> 9, torch.arange(
            nsuper + 1, device=targets.device)).int()

    def query(self, queries):
        return ops.pcd_capped_nn_index(queries, self.tgt, self.ukeys, self.start, self.super_begin,
                                       self.org, self.h, self.sdims, self.box_lo, self.box_hi,
                                       self.cap, self.index)


def _nn_cell(cap, voxel):
    return max(voxel, cap / 16)


def icp_update(moments, origin):
    """Umeyama from the 18 device moments (host, float64) -> 4x4, identity below 3
    correspondences."""
    m = moments.cpu().numpy()
    n = m[0]
    if n < 3:
        return np.eye(4)
    ms, mt = m[2:5] / n, m[5:8] / n
    var = m[8] / n - ms @ ms
    sigma = m[9:18].reshape(3, 3) / n - np.outer(mt, ms)
    o = np.asarray(origin, np.float64)
    return umeyama_from_stats(n, ms + o, mt + o, var, sigma)


def _fit_rmse(moments, n_src):
    m = moments.cpu().numpy()
    cnt = float(m[0])
    return (cnt / n_src if n_src else 0.0), (math.sqrt(m[1] / cnt) if cnt else 0.0), m


def icp(src, tgt, grid, origin, max_iter=ICP_MAX_ITER):
    """Point-to-point ICP with scale from the identity; every iteration transforms the stored
    float32 source by the accumulated T -> (T, iterations, fitness, rmse)."""
    n = src.shape[0]
    T = np.eye(4)
    q = src
    _, idx = grid.query(q)
    mom = ops.tnt_icp_moments(q, grid.targets_all, idx, origin)
    fit, rmse, _ = _fit_rmse(mom, n)
    it = 0
    for _ in range(max_iter):
        T = icp_update(mom, origin) @ T
        q = ops.tnt_transform_crop(src, T)
        _, idx = grid.query(q)
        mom = ops.tnt_icp_moments(q, grid.targets_all, idx, origin)
        f2, r2, _ = _fit_rmse(mom, n)
        it += 1
        conv = abs(f2 - fit) < ICP_CONVERGE and abs(r2 - rmse) < ICP_CONVERGE
        fit, rmse = f2, r2
        if conv:
            break
    return T, it, fit, rmse


STAGES = (("voxel", 1.0, 80.0), ("voxel", 0.5, 20.0), ("uniform", None, 2.0))


def refine(src, gt_cropped, T0, vol, tau, counts, times):
    """The three ICP stages -> (final T, stage dicts)."""
    T = np.asarray(T0, np.float64)
    stages = []
    for k, (method, vfac, dfac) in enumerate(STAGES):
        t0 = _sync_time()
        s = crop(src, vol, T)
        counts[f"stage{k}_source_cropped"] = int(s.shape[0])
        if method == "voxel":
            s, t = voxel_downsample(s, vfac * tau), voxel_downsample(gt_cropped, vfac * tau)
        else:
            s, t = uniform_downsample(s), uniform_downsample(gt_cropped)
        counts[f"stage{k}_source"], counts[f"stage{k}_target"] = int(s.shape[0]), int(t.shape[0])
        d = dfac * tau
        if s.shape[0] == 0 or t.shape[0] == 0:
            Ti, it, fit, rmse = np.eye(4), 0, 0.0, 0.0
        else:
            grid = NNGrid(t, vol.lo, vol.hi, d, _nn_cell(d, (vfac or 0.5) * tau))
            Ti, it, fit, rmse = icp(s, t, grid, vol.centre)
        T = Ti @ T
        stages.append(dict(method=method, max_distance=d, T=T.tolist(), iterations=int(it),
                           fitness=float(fit), rmse=float(rmse)))
        times[f"icp{k}_s"] = _sync_time() - t0
    return T, stages


def curve(d, tau):
    """Cumulative np.histogram of d (device float64) over the edges k tau / 100, k < 500 (the
    last bin closed), divided by len(d)."""
    edges = np.arange(N_EDGES) * tau / 100
    n = d.shape[0]
    if n == 0:
        return np.zeros(N_EDGES - 1)
    ds = torch.sort(d).values
    e = torch.from_numpy(edges).to(d.device)
    below = torch.searchsorted(ds, e[1:], right=False)                   # #(d < e_k+1)
    below[-1] = torch.searchsorted(ds, e[-1:], right=True)[0]            # last bin closed
    first = torch.searchsorted(ds, e[:1], right=False)[0]                # d < e_0 is not counted
    return ((below - first).double() / n).cpu().numpy()


def score(src, gt_cropped, T, vol, tau, counts, times, return_arrays=False):
    t0 = _sync_time()
    s = voxel_downsample(crop(src, vol, T), tau / 2)
    t = voxel_downsample(gt_cropped, tau / 2)
    counts["score_source"], counts["score_target"] = int(s.shape[0]), int(t.shape[0])
    cap = 5 * tau
    dev = src.device
    empty = torch.zeros(0, device=dev, dtype=torch.float64)
    d1 = NNGrid(t, vol.lo, vol.hi, cap, _nn_cell(cap, tau / 2)).query(s)[0] if len(t) else \
        torch.full((s.shape[0],), cap, device=dev, dtype=torch.float64)
    d2 = NNGrid(s, vol.lo, vol.hi, cap, _nn_cell(cap, tau / 2)).query(t)[0] if len(s) else \
        torch.full((t.shape[0],), cap, device=dev, dtype=torch.float64)
    if len(s) and len(t):
        p = int((d1 < tau).sum().item()) / len(d1)
        r = int((d2 < tau).sum().item()) / len(d2)
    else:
        p = r = 0.0
    f = 2 * p * r / (p + r) if p + r > 0 else 0.0
    out = dict(precision=p, recall=r, fscore=f, curve_precision=curve(d1 if len(d1) else empty, tau).tolist(),
               curve_recall=curve(d2 if len(d2) else empty, tau).tolist())
    times["score_s"] = _sync_time() - t0
    if return_arrays:
        out.update(source=s, target=t, d1=d1, d2=d2)
    return out


# ------------------------------------------------------------------------------ one scene
def _load_trajectory(trajectory):
    if isinstance(trajectory, Trajectory):
        return trajectory
    if isinstance(trajectory, (str, os.PathLike)):
        if os.path.isdir(trajectory):
            return trajectory_from_run(trajectory)
        return trajectory_from_log(trajectory)
    raise TypeError("trajectory must be a Trajectory, a run directory or a .log path")


def prepare(trajectory, gt_dir, scene, tau=None, images=None):
    """Host-side checks and readers, before any device work -> (tau, trajectory, paths)."""
    tau = scene_tau(scene, tau)
    paths = gt_paths(gt_dir, scene)
    for k, p in paths.items():
        if not os.path.isfile(p):
            raise FileNotFoundError(f"ground truth {k}: {p}")
    traj = _load_trajectory(trajectory)
    gt_log = read_log(paths["log"])
    pair_cameras(traj, len(gt_log), images)
    return tau, traj, paths, gt_log


def evaluate_scene(points_or_ply, trajectory, gt_dir, scene, tau=None, seed=0, return_arrays=False,
                   images=None, device="cuda:0"):
    """Scores one Tanks and Temples training scene.  `points_or_ply` is a float32 CUDA (N,3)
    tensor or a PLY path; `trajectory` a Trajectory, a run directory (cams/, view_names.txt) or
    a .log.  Returns a dict with precision, recall, fscore, tau, the alignment, every stage's
    transform / iterations / fitness / rmse, point counts, both curves and device-synchronised
    times per phase (time_s).  return_arrays adds the scored device clouds and d1, d2."""
    tau, traj, paths, gt_log = prepare(trajectory, gt_dir, scene, tau, images)
    times = {}
    t0 = time.perf_counter()
    trans = read_trans(paths["trans"])
    vol_args = read_crop(paths["crop"])
    if isinstance(points_or_ply, (str, os.PathLike)):
        dev = torch.device(device)
        if dev.type != "cuda" or not torch.cuda.is_available():
            raise _lib.CasMVSError("Tanks and Temples scoring runs on the GPU (no CPU fallback)")
        src = torch.from_numpy(read_points(points_or_ply)).to(dev)
    elif torch.is_tensor(points_or_ply) and points_or_ply.is_cuda:
        src = points_or_ply
        if src.dtype != torch.float32 or src.dim() != 2 or src.shape[1] != 3:
            raise ValueError("points must be a float32 CUDA tensor of shape (N,3)")
        src = src.contiguous()
    else:
        raise TypeError("points must be a CUDA (N,3) tensor or a PLY path")
    with torch.cuda.device(src.device):
        gt = torch.from_numpy(read_points(paths["ply"])).to(src.device)
        vol = CropVolume(*vol_args, src.device)
        times["load_s"] = _sync_time() - t0
        t1 = time.perf_counter()
        T0, al = align(traj, gt_log[:, :3, 3], trans, images, seed)
        times["align_s"] = time.perf_counter() - t1
        t2 = _sync_time()
        gt_c = crop(gt, vol)
        counts = dict(source=int(src.shape[0]), target=int(gt.shape[0]),
                      target_cropped=int(gt_c.shape[0]))
        times["crop_gt_s"] = _sync_time() - t2
        T, stages = refine(src, gt_c, T0, vol, tau, counts, times)
        sc = score(src, gt_c, T, vol, tau, counts, times, return_arrays)
    times["total_s"] = time.perf_counter() - t0
    out = dict(scene=scene, tau=tau, seed=int(seed), precision=sc.pop("precision"),
               recall=sc.pop("recall"), fscore=sc.pop("fscore"), alignment=dict(al, T0=T0.tolist()),
               stages=stages, T=T.tolist(), counts=counts, time_s=times)
    out.update(sc)
    return out


def evaluate_mesh(mesh, trajectory, gt_dir, scene, tau=None, seed=0, images=None, device="cuda:0",
                  return_arrays=False):
    """Scores a mesh of one Tanks and Temples training scene: its surface is sampled at tau / 4
    (mesh_sample.sample_surface), below the tau / 2 voxels scoring downsamples to, so every voxel
    the surface crosses gets samples, and the samples are scored by evaluate_scene.  `mesh` is
    (verts (V,3) float32, faces (F,3) int) CUDA tensors or a mesh PLY path.  Returns
    evaluate_scene's dict plus n_faces, n_samples, spacing and time_s["sample_s"];
    return_arrays adds the samples."""
    from . import mesh_sample
    tau = scene_tau(scene, tau)
    prepare(trajectory, gt_dir, scene, tau, images)
    verts, faces = mesh_sample.load_mesh(mesh, device)
    t0 = _sync_time()
    samples = mesh_sample.sample_surface(verts, faces, tau / 4)
    t1 = _sync_time()
    out = evaluate_scene(samples, trajectory, gt_dir, scene, tau, seed, return_arrays, images)
    out.update(n_faces=int(len(faces)), n_samples=int(len(samples)), spacing=tau / 4)
    out["time_s"]["sample_s"] = t1 - t0
    if return_arrays:
        out["samples"] = samples
    return out


def _fmt(r):
    t = r["time_s"]
    return (f"{r['scene']}: tau {r['tau']:g}  precision {r['precision']:.4f}  recall "
            f"{r['recall']:.4f}  F {r['fscore']:.4f}  ({r['alignment']['inliers']}/"
            f"{r['alignment']['pairs']} camera inliers)  time: "
            + " ".join(f"{k[:-2]} {v:.3f}s" for k, v in t.items() if k.endswith("_s")))


def write_json(path, result):
    keep = {k: v for k, v in result.items() if not torch.is_tensor(v)}
    with open(path, "w") as f:
        json.dump(keep, f, indent=1)


def main(argv=None):
    ap = argparse.ArgumentParser(description="Score a reconstruction of a Tanks and Temples "
                                             "training scene on the GPU.")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--ply", help="the reconstruction's point cloud")
    src.add_argument("--mesh", help="a mesh PLY: its surface is sampled at tau / 4 and scored "
                                    "like points")
    g = ap.add_mutually_exclusive_group(required=True)
    g.add_argument("--run_dir", help="a run's scan directory: cams/*_cam.txt and view_names.txt")
    g.add_argument("--log", help="the reconstruction's camera poses as a .log")
    ap.add_argument("--gt_dir", required=True)
    ap.add_argument("--scene", required=True)
    ap.add_argument("--images", default=None,
                    help="the complete image directory: pair cameras by image name")
    ap.add_argument("--tau", type=float, default=None)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--out", default="")
    a = ap.parse_args(argv)
    try:
        prepare(a.run_dir or a.log, a.gt_dir, a.scene, a.tau, a.images)
    except (ValueError, FileNotFoundError) as e:
        raise SystemExit(f"tnt_eval: {e}")
    if a.mesh:
        r = evaluate_mesh(a.mesh, a.run_dir or a.log, a.gt_dir, a.scene, a.tau, a.seed,
                          images=a.images, device=a.device)
    else:
        r = evaluate_scene(a.ply, a.run_dir or a.log, a.gt_dir, a.scene, a.tau, a.seed,
                           images=a.images, device=a.device)
    print(_fmt(r), flush=True)
    if a.out:
        write_json(a.out, r)
    return r


if __name__ == "__main__":
    main()
