"""float64 numpy / scipy restatement of the reference's DTU scorer, the test oracle of
casmvsnet_pl_b200/dtu_eval.py (paths relative to the reference root):

    thin            evaluations/dtu/reducePts_haa.m:9-33 (randperm order, rangesearch <= dst,
                    visited-and-not-removed points are kept), called at PointCompareMain.m:7 with
                    dst = 0.2 (BaseEvalMain_web.m:25); visited sequentially here
    capped_nn       MaxDistCP.m:3 (60 everywhere first), :5-18 (blocks of MaxDist from BB(1,:),
                    Low <= q < High), :20-33 (nearest neighbour among targets within MaxDist of the
                    block); MaxDist = 60 at PointCompareMain.m:20
    data_in_mask    PointCompareMain.m:32-41
    stl_above_plane PointCompareMain.m:53
    stats           BaseEvalMain_web.m:59-68, ComputeStat_web.m:49-65 (mean / median / var)

The visiting order is the engine's: torch.randperm(n) with a CPU generator seeded by `seed`.
The "<= dst" predicate is (dx*dx + dy*dy) + dz*dz <= dst*dst in float64 on the float32 values.
Distances are min(nearest-neighbour distance, 60) inside the block grid: the MATLAB's value
whenever that is below 60 (it can report more than 60 near block faces, which no statistic reads).
"""
from __future__ import annotations

import numpy as np
import torch
from scipy.spatial import cKDTree


def visiting_order(n, seed):
    """RandOrd of reducePts_haa.m:9, seeded: the k-th visited point."""
    return torch.randperm(n, generator=torch.Generator().manual_seed(int(seed))).numpy()


def within(a, b, dst):
    """|a - b| <= dst, row-wise, in float64 with the engine's operation order."""
    d = np.asarray(a, np.float32).astype(np.float64) - np.asarray(b, np.float32).astype(np.float64)
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2] <= dst * dst


def neighbour_lists(pts, dst):
    """CSR (offsets, nbrs) of the '<= dst' graph (no self loops)."""
    pts = np.asarray(pts, np.float32)
    n = len(pts)
    pairs = cKDTree(pts.astype(np.float64)).query_pairs(dst * (1 + 1e-6) + 1e-9,
                                                        output_type="ndarray")
    pairs = pairs[within(pts[pairs[:, 0]], pts[pairs[:, 1]], dst)] if len(pairs) else pairs
    src = np.concatenate([pairs[:, 0], pairs[:, 1]]) if len(pairs) else np.zeros(0, np.int64)
    dst_ = np.concatenate([pairs[:, 1], pairs[:, 0]]) if len(pairs) else np.zeros(0, np.int64)
    order = np.argsort(src, kind="stable")
    offs = np.zeros(n + 1, np.int64)
    np.add.at(offs, src + 1, 1)
    return np.cumsum(offs), dst_[order]


def thin(pts, dst=0.2, seed=0):
    """reducePts_haa.m sequentially -> ascending indices of the kept points."""
    n = len(pts)
    if n == 0:
        return np.zeros(0, np.int64)
    offs, nbrs = neighbour_lists(pts, dst)
    keep = np.ones(n, bool)
    for i in visiting_order(n, seed):                # reducePts_haa.m:25-31
        if keep[i]:
            keep[nbrs[offs[i]:offs[i + 1]]] = False
    return np.nonzero(keep)[0]


def block_grid(bb, max_dist=60.0):
    """Outer faces of MaxDistCP.m's blocks: Low = BB1 + 0*MaxDist, last High =
    (BB1 + Range*MaxDist) + MaxDist."""
    bb = np.asarray(bb, np.float64).reshape(2, 3)
    rng = np.floor((bb[1] - bb[0]) / max_dist)
    return bb[0] + 0.0 * max_dist, (bb[0] + rng * max_dist) + max_dist


def capped_nn(queries, targets, bb, max_dist=60.0):
    q = np.asarray(queries, np.float32).astype(np.float64)
    t = np.asarray(targets, np.float32).astype(np.float64)
    out = np.full(len(q), max_dist)
    lo, hi = block_grid(bb, max_dist)
    inside = np.all((q >= lo) & (q < hi), axis=1) if len(q) else np.zeros(0, bool)
    if len(t) and inside.any():
        d, _ = cKDTree(t).query(q[inside], k=1, distance_upper_bound=max_dist)
        out[inside] = np.minimum(d, max_dist)
    return out


def matlab_round(x):
    """MATLAB round: halves away from zero."""
    x = np.asarray(x, np.float64)
    t = np.trunc(x)
    return t + np.sign(x) * (np.abs(x - t) >= 0.5)


def data_in_mask(pts, obs_mask, bb, res):
    p = np.asarray(pts, np.float32).astype(np.float64)
    b1 = np.asarray(bb, np.float64).reshape(2, 3)[0]
    v = matlab_round((p - b1) / res + 1)
    size = np.array(obs_mask.shape)
    inside = np.all((v >= 1) & (v <= size), axis=1)
    out = np.zeros(len(p), bool)
    idx = (v[inside] - 1).astype(np.int64)
    out[inside] = np.asarray(obs_mask, bool)[idx[:, 0], idx[:, 1], idx[:, 2]]
    return out


def stl_above_plane(pts, P):
    p = np.asarray(pts, np.float32).astype(np.float64)
    P = np.asarray(P, np.float64).reshape(4)
    return ((P[0] * p[:, 0] + P[1] * p[:, 1]) + P[2] * p[:, 2]) + P[3] > 0


def stats(d, sel, max_dist=20.0):
    """MATLAB mean / median / var (unbiased; 0 for one value; NaN for none) and the count."""
    x = np.asarray(d, np.float64)[np.asarray(sel, bool) & (np.asarray(d) < max_dist)]
    if len(x) == 0:
        return dict(mean=np.nan, median=np.nan, var=np.nan, n=0)
    return dict(mean=float(x.mean()), median=float(np.median(x)),
                var=float(x.var(ddof=1)) if len(x) > 1 else 0.0, n=len(x))


def evaluate(data, stl, obs_mask, bb, res, plane, dst=0.2, seed=0):
    """PointCompareMain.m + the statistics of one scan."""
    kept = thin(data, dst, seed)
    q = np.asarray(data, np.float32)[kept]
    d_data = capped_nn(q, stl, bb)
    d_stl = capped_nn(stl, q, bb)
    in_mask = data_in_mask(q, obs_mask, bb, res)
    above = stl_above_plane(stl, plane)
    acc, comp = stats(d_data, in_mask), stats(d_stl, above)
    return dict(kept=kept, Ddata=d_data, Dstl=d_stl, data_in_mask=in_mask, stl_above_plane=above,
                acc=acc, comp=comp, overall=(acc["mean"] + comp["mean"]) / 2)
