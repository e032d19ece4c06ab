"""float64 numpy / scipy restatement of the Tanks and Temples training-set scoring of
casmvsnet_pl_b200/tnt_eval.py (steps 2 and 3 of its protocol: the three ICP refinements and the
scores), the test oracle of csrc/tnt_eval.cu and of the index-returning nearest-neighbour search
of csrc/pcd_eval.cu.

Every expression is written in the operation order the kernels use (include/casmvs.h), so that
crops, downsampled points and nearest-neighbour distances and indices agree bit for bit:

    transform      x' = float32(((T00 x + T01 y) + T02 z) + T03), likewise y', z'
    crop           Open3D CropInPolygon on the float32 point, in double
    voxel mean     per voxel, per axis: sequential double sum in input order / count -> float32
    nearest        d^2 = (dx*dx + dy*dy) + dz*dz, dx = t - q, in double; the lowest original index
                   wins an exact tie; no correspondence unless d^2 < cap^2

Nearest neighbours come from scipy's cKDTree; its candidates are re-ranked with the exact
expression above, widening the candidate list while a tie could reach past it.  Umeyama is taken
from the correspondences with two-pass means (the product sums moments on the device), so an ICP
update agrees with the product's to rounding, not bit for bit.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

MAX_ITER = 20
CONVERGE = 1e-6
UNIFORM_MAX = 4_000_000
N_EDGES = 500


# ------------------------------------------------------------------------------ point operations
def transform(pts, T):
    """float32(T p) in double, rows ((T0 x + T1 y) + T2 z) + T3."""
    p = np.asarray(pts, np.float32).astype(np.float64)
    T = np.asarray(T, np.float64).reshape(4, 4)
    out = np.empty((len(p), 3), np.float32)
    for r in range(3):
        out[:, r] = (((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3]).astype(np.float32)
    return out


def plane_axes(axis):
    return {0: (1, 2), 1: (0, 2), 2: (0, 1)}[axis]


def crop_mask(pts, axis, axis_min, axis_max, polygon_uv):
    """Open3D SelectionPolygonVolume::CropInPolygon on float32 points, in double."""
    p = np.asarray(pts, np.float32).astype(np.float64)
    poly = np.asarray(polygon_uv, np.float64).reshape(-1, 2)
    u, v = plane_axes(axis)
    pa, pu, pv = p[:, axis], p[:, u], p[:, v]
    keep = (pa >= axis_min) & (pa <= axis_max)
    below = np.zeros(len(p), np.int64)
    m = len(poly)
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(m):
            j = (i + 1) % m
            iu, iv, ju, jv = poly[i, 0], poly[i, 1], poly[j, 0], poly[j, 1]
            cross = ((iu < pu) & (ju >= pu)) | ((ju < pu) & (iu >= pu))
            node = iv + ((pu - iu) / (ju - iu)) * (jv - iv)
            below += cross & (node < pv)
    return keep & (below % 2 == 1)


def voxel_grid(pts, voxel):
    """(origin, dims, integer voxel coordinates (N,3)) of the voxel downsampling."""
    p = np.asarray(pts, np.float32).astype(np.float64)
    origin = p.min(0) - voxel * 0.5
    ijk = np.floor((p - origin) / voxel)
    dims = np.floor((p.max(0) - origin) / voxel).astype(np.int64) + 1
    return origin, dims, ijk.astype(np.int64)


def voxel_downsample(pts, voxel):
    """One point per occupied voxel in ascending (ix, iy, iz) order: the float32 mean of its
    points, summed in double in input order."""
    p32 = np.asarray(pts, np.float32)
    if len(p32) == 0:
        return np.zeros((0, 3), np.float32)
    _, dims, ijk = voxel_grid(p32, voxel)
    key = (ijk[:, 0] * dims[1] + ijk[:, 1]) * dims[2] + ijk[:, 2]
    order = np.argsort(key, kind="stable")
    ks = key[order]
    first = np.r_[True, ks[1:] != ks[:-1]]
    vid = np.cumsum(first) - 1
    starts = np.nonzero(first)[0]
    rank = np.arange(len(ks)) - starts[vid]
    nv = len(starts)
    sums = np.zeros((nv, 3))
    counts = np.bincount(vid, minlength=nv).astype(np.float64)
    p = p32.astype(np.float64)[order]
    for r in range(int(rank.max()) + 1):       # the r-th point of every voxel: input order
        sel = rank == r
        sums[vid[sel]] = sums[vid[sel]] + p[sel]
    return (sums / counts[:, None]).astype(np.float32)


def uniform_downsample(pts, max_points=UNIFORM_MAX):
    n = len(pts)
    if n <= max_points:
        return np.asarray(pts, np.float32)
    k = int(round(n / max_points))
    return np.asarray(pts, np.float32)[::k]


def exact_d2(q, t):
    d = np.asarray(t, np.float32).astype(np.float64) - np.asarray(q, np.float32).astype(np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def nearest(queries, targets, cap):
    """(dist float64, index int64) of each query's nearest target strictly closer than cap, with
    ties to the lower index; (cap, -1) when there is none."""
    q = np.asarray(queries, np.float32)
    t = np.asarray(targets, np.float32)
    dist = np.full(len(q), float(cap))
    index = np.full(len(q), -1, np.int64)
    if len(q) == 0 or len(t) == 0:
        return dist, index
    tree = cKDTree(t.astype(np.float64))
    todo = np.arange(len(q))
    k = 8
    cap2 = cap * cap
    while len(todo):
        kk = min(k, len(t))
        _, nb = tree.query(q[todo].astype(np.float64), k=kk, distance_upper_bound=cap * (1 + 1e-9) + 1e-12)
        nb = nb.reshape(len(todo), kk)
        valid = nb < len(t)
        d2 = np.where(valid, exact_d2(q[todo][:, None, :], t[np.minimum(nb, len(t) - 1)]), np.inf)
        best = d2.min(1)
        # a tie (or a candidate kd-rounding put later) could lie past the k-th: widen and retry
        last = d2[:, -1]
        again = valid[:, -1] & (last <= best * (1 + 1e-9) + 1e-300) & (kk < len(t))
        done = ~again
        rows = todo[done]
        b = best[done]
        idx = np.where(d2[done] == b[:, None], np.where(valid[done], nb[done], np.iinfo(np.int64).max),
                       np.iinfo(np.int64).max).min(1)
        ok = b < cap2
        dist[rows[ok]] = np.sqrt(b[ok])
        index[rows[ok]] = idx[ok]
        todo = todo[again]
        k *= 4
    return dist, index


# ------------------------------------------------------------------------------ registration
def umeyama(src, dst):
    """4x4 similarity dst ~ c R src + t (Umeyama with scale), from point arrays."""
    s = np.asarray(src, np.float64)
    d = np.asarray(dst, np.float64)
    ms, md = s.mean(0), d.mean(0)
    sc, dc = s - ms, d - md
    var = (sc * sc).sum(1).mean()
    sigma = dc.T @ sc / len(s)
    U, D, Vt = np.linalg.svd(sigma)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1
    R = U @ np.diag(S) @ Vt
    c = (D * S).sum() / var
    T = np.eye(4)
    T[:3, :3] = c * R
    T[:3, 3] = md - c * R @ ms
    return T


def icp_scores(q, tgt, idx, dist):
    n = int((idx >= 0).sum())
    fit = n / len(q) if len(q) else 0.0
    rmse = float(np.sqrt((dist[idx >= 0] ** 2).sum() / n)) if n else 0.0
    return fit, rmse


def icp(src, tgt, max_dist, max_iter=MAX_ITER):
    """Point-to-point ICP with scale from the identity -> (T, iterations, fitness, rmse)."""
    src = np.asarray(src, np.float32)
    T = np.eye(4)
    dist, idx = nearest(src, tgt, max_dist)
    fit, rmse = icp_scores(src, tgt, idx, dist)
    it = 0
    for _ in range(max_iter):
        q = transform(src, T)
        sel = idx >= 0
        upd = umeyama(q[sel], np.asarray(tgt, np.float32)[idx[sel]]) if sel.sum() >= 3 else np.eye(4)
        T = upd @ T
        q = transform(src, T)
        dist, idx = nearest(q, tgt, max_dist)
        f2, r2 = icp_scores(q, tgt, idx, dist)
        it += 1
        conv = abs(f2 - fit) < CONVERGE and abs(r2 - rmse) < CONVERGE
        fit, rmse = f2, r2
        if conv:
            break
    return T, it, fit, rmse


def crop(pts, crop_vol):
    axis, amin, amax, poly = crop_vol
    p = np.asarray(pts, np.float32)
    return p[crop_mask(p, axis, amin, amax, poly)]


def stage_clouds(src, gt, T_init, crop_vol, method, voxel=None):
    s = crop(transform(src, T_init), crop_vol)
    t = crop(gt, crop_vol)
    if method == "voxel":
        return voxel_downsample(s, voxel), voxel_downsample(t, voxel)
    return uniform_downsample(s), uniform_downsample(t)


def refine(src, gt, T0, crop_vol, tau):
    """The three ICP stages -> (final T, [(T, iterations, fitness, rmse)])."""
    T = np.asarray(T0, np.float64)
    stages = []
    for method, voxel, d in (("voxel", tau, 80 * tau), ("voxel", tau / 2, 20 * tau), ("uniform", None, 2 * tau)):
        s, t = stage_clouds(src, gt, T, crop_vol, method, voxel)
        Ti, it, fit, rmse = icp(s, t, d)
        T = Ti @ T
        stages.append((T.copy(), it, fit, rmse))
    return T, stages


def curve(d, tau):
    """Cumulative np.histogram over edges k tau / 100 (k < 500) divided by len(d)."""
    edges = np.arange(N_EDGES) * tau / 100
    if len(d) == 0:
        return np.zeros(N_EDGES - 1)
    h, _ = np.histogram(d, edges)
    return np.cumsum(h) / len(d)


def scores(src, gt, T, crop_vol, tau):
    s = voxel_downsample(crop(transform(src, T), crop_vol), tau / 2)
    t = voxel_downsample(crop(gt, crop_vol), tau / 2)
    d1, _ = nearest(s, t, 5 * tau)
    d2, _ = nearest(t, s, 5 * tau)
    p = float((d1 < tau).sum() / len(d1)) if len(d1) and len(d2) else 0.0
    r = float((d2 < tau).sum() / len(d2)) if len(d1) and len(d2) else 0.0
    f = 2 * p * r / (p + r) if p + r > 0 else 0.0
    return dict(precision=p, recall=r, fscore=f, d1=d1, d2=d2, curve_precision=curve(d1, tau),
                curve_recall=curve(d2, tau), n_source=len(s), n_target=len(t))


def evaluate(src, gt, T0, crop_vol, tau):
    T, stages = refine(src, gt, T0, crop_vol, tau)
    out = scores(src, gt, T, crop_vol, tau)
    out.update(T=T, stages=stages)
    return out
