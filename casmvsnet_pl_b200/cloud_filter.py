"""Statistical outlier removal for fused point clouds on the GPU (csrc/pcd_eval.cu; numpy float64
restatement in oracle/cloud_filter_oracle.py, bit for bit).

    keep, stats = remove_statistical_outliers(xyz, k=20, std_ratio=2.0)

    python -m casmvsnet_pl_b200.cloud_filter --ply in.ply --out out.ply [--neighbours 20]
                                             [--std_ratio 2.0]

The rule, for N float32 points, k in 1..64 and a ratio r > 0 (include/casmvs.h states every
operation):
1. d(i, j) = sqrt((dx*dx + dy*dy) + dz*dz) in double, dx = double(x_j) - double(x_i), every
   operation rounded to nearest;
2. m_i is the mean of the k smallest d(i, j) over j != i: the point is not its own neighbour, but
   exact duplicates of it are, at distance 0.  The k distances are summed left to right in
   ascending order, then divided by k;
3. mu = sum m_i / N and sigma = sqrt(sum (m_i - mu)^2 / (N - 1)), each sum in double over chunks
   of STAT_CHUNK points in input order, left to right, then the chunk sums left to right;
4. point i is kept when m_i <= mu + r sigma.  <= keeps every point of a cloud whose m_i are all
   equal (sigma = 0, a regular lattice).
The kept points keep their input order; two runs give the same bits.  The rule is modelled on
Open3D's remove_statistical_outlier(nb_neighbors, std_ratio); agreement with it is not checked.

The k nearest neighbours are searched exactly on a grid of cells grouped in super cells of 8^3
(dtu_eval's layout).  The cell edge is chosen so that occupied cells hold about k points: it
starts from a bounding-box cube of N / k cells and shrinks while the occupied cells hold more than
2k points on average (surfaces and clusters fill few of a box's cells).  The search is exact for
any edge; the edge only sets its speed."""
from __future__ import annotations

import argparse
import math
import time

import numpy as np
import torch

from . import _lib, io, mesh, ops

DEFAULT_K = 20
DEFAULT_STD_RATIO = 2.0
MAX_K = 64
STAT_CHUNK = 1024
# device bytes per point: the keys and their sort, the sorted points, the cell lists, the mean
# distances, the mask and the compaction.  bench_cloud_filter.py measured a peak of 63.2 to 64.2
# bytes per point above the input cloud (34.2 M and 103.3 M points, k = 20 and 64) on an H100
BYTES_PER_POINT = 72
GRID_TRIALS = 4           # cell edges tried before the search runs on the last one
MAX_SUPER = 256           # super cells per axis at most (the capped_nn grid's bound)
_OUTSIDE = torch.iinfo(torch.int64).max


def _sync_time():
    torch.cuda.synchronize()
    return time.perf_counter()


def check_options(k, std_ratio):
    """Raises ValueError unless k is an integer in 1..MAX_K and std_ratio a finite number > 0."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= MAX_K:
        raise ValueError(f"k must be an integer in 1..{MAX_K}, got {k!r}")
    if isinstance(std_ratio, bool) or not isinstance(std_ratio, (int, float, np.integer, np.floating)) \
            or not (math.isfinite(std_ratio) and std_ratio > 0):
        raise ValueError(f"std_ratio must be a finite number > 0, got {std_ratio!r}")


def _check_inputs(xyz, k, std_ratio, max_bytes):
    check_options(k, std_ratio)
    if not (torch.is_tensor(xyz) and xyz.dim() == 2 and xyz.shape[1] == 3):
        got = tuple(xyz.shape) if torch.is_tensor(xyz) else type(xyz).__name__
        raise ValueError(f"xyz must be a float32 CUDA tensor of shape (N, 3), got {got}")
    n = xyz.shape[0]
    if not k < n < 2 ** 31:
        raise ValueError(f"a cloud of {n} points cannot be filtered with k = {k}: it needs more "
                         f"than k and fewer than 2^31 points")
    if not (xyz.is_cuda and xyz.dtype == torch.float32):
        raise ValueError(f"xyz must be a float32 CUDA tensor of shape (N, 3), got {xyz.dtype} "
                         f"on {xyz.device}")
    need = n * BYTES_PER_POINT
    budget = mesh.device_budget(xyz.device, max_bytes)
    if need > budget:
        raise _lib.CasMVSError(f"filtering {n} points needs {need} bytes of device memory but "
                               f"{max(budget, 0)} bytes are available")
    bad = ~torch.isfinite(xyz).all(1)
    if bool(bad.any()):
        raise ValueError(f"xyz holds a non-finite coordinate at point {int(bad.nonzero()[0, 0])}")


def _cells(keys_sorted):
    ukeys, counts = torch.unique_consecutive(keys_sorted, return_counts=True)
    start = torch.zeros(len(ukeys) + 1, device=keys_sorted.device, dtype=torch.int32)
    torch.cumsum(counts, 0, out=start[1:])
    return ukeys, start


def _grid(pts, k, times):
    """The search grid: the cloud binned and key-sorted at the chosen cell edge."""
    t0 = _sync_time()
    lo = pts.min(0).values.double().cpu().numpy()
    hi = pts.max(0).values.double().cpu().numpy()
    ext = hi - lo
    emax = float(ext.max())
    n = pts.shape[0]
    t1 = _sync_time()
    times["bounds_keys_s"] = t1 - t0
    times["sort_cells_s"] = 0.0
    if emax == 0.0:
        h = h_min = 1.0                                      # every point in one cell
    else:
        h_min = emax / (8 * (MAX_SUPER - 1))
        h = max(emax * (k / n) ** (1 / 3), h_min)
    for trial in range(GRID_TRIALS):
        t1 = _sync_time()
        sdims = [int(math.floor(e / (8 * h))) + 2 for e in ext]
        keys = ops.pcd_cell_keys(pts, lo, h, [8 * s for s in sdims], sub=8)
        t2 = _sync_time()
        keys, order = torch.sort(keys)
        ukeys, start = _cells(keys)
        t3 = _sync_time()
        times["bounds_keys_s"] += t2 - t1
        times["sort_cells_s"] += t3 - t2
        occupancy = n / len(ukeys)
        if occupancy <= 2 * k or h <= h_min or trial + 1 == GRID_TRIALS:
            break
        h = max(h * math.sqrt(k / occupancy), h_min)        # surfaces: occupancy ~ h^2
    if int(keys[-1]) == _OUTSIDE:
        raise _lib.CasMVSError("cloud_filter: a point fell outside its own bounding-box grid")
    t3 = _sync_time()
    nsuper = sdims[0] * sdims[1] * sdims[2]
    super_begin = torch.searchsorted(ukeys >> 9, torch.arange(nsuper + 1, device=pts.device)).int()
    # widening of the pruning boxes: far above the rounding of keys and bounds at these coordinates
    pad = 2.0 ** -30 * (float(np.abs(lo).max()) + float(np.abs(hi).max()) + 16 * h)
    times["sort_cells_s"] += _sync_time() - t3
    return dict(lo=lo, h=h, sdims=sdims, pad=pad, order=order, ukeys=ukeys, start=start,
                super_begin=super_begin, cells=len(ukeys), trials=trial + 1)


def _mean_distance(pts, k, times):
    g = _grid(pts, k, times)
    t0 = _sync_time()
    m = ops.pcd_knn_mean(pts[g["order"]].contiguous(), k, g["ukeys"], g["start"], g["super_begin"],
                         g["lo"], g["h"], g["sdims"], g["pad"], g["order"])
    times["search_s"] = _sync_time() - t0
    return m, g


def mean_neighbour_distance(xyz, k=DEFAULT_K, max_bytes=None):
    """m_i, the mean distance of every point of xyz ((N,3) float32 CUDA) to its k nearest other
    points, as (N,) float64 on the device (steps 1-2 of the rule)."""
    _check_inputs(xyz, k, 1.0, max_bytes)
    with torch.cuda.device(xyz.device):
        return _mean_distance(xyz.contiguous(), int(k), {})[0]


def _filter(xyz, k, std_ratio):
    pts = xyz.contiguous()
    times = {}
    m, g = _mean_distance(pts, int(k), times)
    t0 = _sync_time()
    st, mask, counts, _ = ops.pcd_sor_keep(m, float(std_ratio))
    mu, sigma, thr = st.tolist()
    kept = int(counts.sum())
    times["statistics_s"] = _sync_time() - t0
    stats = dict(points=pts.shape[0], kept=kept, k=int(k), std_ratio=float(std_ratio), mean=mu,
                 std=sigma, threshold=thr, cell=g["h"], cells=g["cells"], grid_trials=g["trials"],
                 time_s=times)
    return pts, mask, counts, stats


def remove_statistical_outliers(xyz, k=DEFAULT_K, std_ratio=DEFAULT_STD_RATIO, max_bytes=None):
    """Statistical outlier removal of xyz ((N,3) float32 CUDA tensor) -> (keep (N,) bool CUDA
    tensor, stats: points, kept, k, std_ratio, mean, std, threshold, cell, cells, grid_trials and
    time_s per phase).  Raises ValueError on bad options or input (k outside 1..64, std_ratio not
    finite and > 0, N <= k, a non-finite point) and CasMVSError when the work would not fit in
    mesh.device_budget (BYTES_PER_POINT per point; max_bytes overrides the budget)."""
    _check_inputs(xyz, k, std_ratio, max_bytes)
    with torch.cuda.device(xyz.device):
        _, mask, _, stats = _filter(xyz, k, std_ratio)
    return mask.bool(), stats


def filter_points(xyz, k=DEFAULT_K, std_ratio=DEFAULT_STD_RATIO, max_bytes=None):
    """remove_statistical_outliers applied: -> (the kept points (M,3) float32 in input order,
    their input indices (M,) int64, stats)."""
    _check_inputs(xyz, k, std_ratio, max_bytes)
    with torch.cuda.device(xyz.device):
        pts, mask, counts, stats = _filter(xyz, k, std_ratio)
        kept, index = ops.tnt_compact(pts, mask, counts)
    return kept, index, stats


def summary(st):
    """One line of the stats."""
    return (f"kept {st['kept']} of {st['points']} points (k {st['k']}, std ratio "
            f"{st['std_ratio']:g}: mean distance {st['mean']:.6g}, std {st['std']:.6g}, threshold "
            f"{st['threshold']:.6g})")


# ------------------------------------------------------------------------------ PLY
_PLY_NAMES = {"i1": "char", "u1": "uchar", "i2": "short", "u2": "ushort", "i4": "int", "u4": "uint",
              "f4": "float", "f8": "double"}


def write_vertices(path, vertices):
    """A binary little-endian PLY of a structured vertex array (as io.read_ply returns it), every
    property in its order and type.  For the fields x y z red green blue it writes the bytes
    fusion.write_ply writes."""
    names = vertices.dtype.names
    if not names:
        raise ValueError("vertices must be a structured array")
    fields = []
    for name in names:
        t = vertices.dtype[name]
        key = f"{t.kind}{t.itemsize}"
        if key not in _PLY_NAMES or t.shape:
            raise ValueError(f"vertex property {name!r} has no PLY scalar type ({t})")
        fields.append((name, "<" + key, _PLY_NAMES[key]))
    out = np.empty(len(vertices), dtype=[(nm, dt) for nm, dt, _ in fields])
    for nm, _, _ in fields:
        out[nm] = vertices[nm]
    header = ("ply\nformat binary_little_endian 1.0\n" f"element vertex {len(out)}\n"
              + "".join(f"property {pn} {nm}\n" for nm, _, pn in fields) + "end_header\n")
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        out.tofile(f)


def _parser():
    ap = argparse.ArgumentParser(description="Remove statistical outliers from a point-cloud PLY "
                                             "on the GPU.")
    ap.add_argument("--ply", required=True, help="the cloud to filter (a PLY with x, y, z)")
    ap.add_argument("--out", required=True, help="the filtered cloud PLY to write, with every "
                                                 "vertex property of the input")
    ap.add_argument("--neighbours", type=int, default=DEFAULT_K,
                    help=f"neighbours per point, 1..{MAX_K} (default {DEFAULT_K})")
    ap.add_argument("--std_ratio", type=float, default=DEFAULT_STD_RATIO,
                    help="drop points whose mean neighbour distance exceeds the cloud's mean by "
                         f"more than this many standard deviations (> 0, default {DEFAULT_STD_RATIO})")
    return ap


def main(argv=None):
    a = _parser().parse_args(argv)
    v = io.read_ply(a.ply)
    if not all(c in (v.dtype.names or ()) for c in "xyz"):
        raise SystemExit(f"{a.ply}: the vertices have no x, y, z")
    xyz = np.ascontiguousarray(np.stack([v["x"], v["y"], v["z"]], axis=1), dtype=np.float32)
    dev = torch.device("cuda", torch.cuda.current_device())
    _, index, st = filter_points(torch.from_numpy(xyz).to(dev), a.neighbours, a.std_ratio)
    write_vertices(a.out, v[index.cpu().numpy()])
    print(f"{a.ply}: {summary(st)}; wrote {a.out}")
    return st


if __name__ == "__main__":
    main()
