"""Float64 numpy restatement of statistical outlier removal (casmvsnet_pl_b200/cloud_filter.py),
bit for bit.

Candidates come from scipy's cKDTree (the k + 1 + MARGIN nearest by its own arithmetic); every
distance is then recomputed by the rule, ((dx*dx + dy*dy) + dz*dz) in double with dx = double(x_j)
- double(x_i), sorted, and the k smallest after the point itself are summed left to right.  The
multiset of the k smallest distances is unique, so it does not matter which of several tied
points the tree returns.  brute_mean_distance is the O(N^2) statement the tests hold it to."""
from __future__ import annotations

import math

import numpy as np

MARGIN = 8
CHUNK = 1024          # cloud_filter.STAT_CHUNK
ROWS = 1 << 16        # query rows per block, to bound host memory


def _d2(p, q):
    """Squared distances in the rule's order: p (..., 3), q (..., 3) float64."""
    dx = q[..., 0] - p[..., 0]
    dy = q[..., 1] - p[..., 1]
    dz = q[..., 2] - p[..., 2]
    return (dx * dx + dy * dy) + dz * dz


def _mean_of_smallest(d2, k):
    """Rows of squared distances (self removed) -> the mean of each row's k smallest distances,
    summed left to right in ascending order."""
    d = np.sqrt(np.sort(d2, axis=1)[:, :k])
    s = np.zeros(len(d))
    for j in range(k):
        s = s + d[:, j]
    return s / k


def mean_distance(xyz, k):
    """m_i of every point of xyz ((N,3) float32) -> (N,) float64."""
    from scipy.spatial import cKDTree
    p = np.asarray(xyz, np.float32).astype(np.float64)
    n = len(p)
    if not 1 <= k < n:
        raise ValueError(f"need 1 <= k < N, got k = {k}, N = {n}")
    kk = min(n, k + 1 + MARGIN)
    tree = cKDTree(p)
    out = np.empty(n)
    for r0 in range(0, n, ROWS):
        rows = np.arange(r0, min(n, r0 + ROWS))
        _, idx = tree.query(p[rows], kk)
        idx = idx.reshape(len(rows), kk)
        d2 = _d2(p[rows][:, None, :], p[idx])
        d2[idx == rows[:, None]] = np.inf                  # the point is not its own neighbour
        # the tree may have returned a duplicate in place of the point itself: then one column
        # too many stays, which the sort puts last (no more than kk - 1 > k are needed)
        out[rows] = _mean_of_smallest(d2, k)
    return out


def brute_mean_distance(xyz, k):
    """mean_distance from all N^2 distances."""
    p = np.asarray(xyz, np.float32).astype(np.float64)
    d2 = _d2(p[:, None, :], p[None, :, :])
    np.fill_diagonal(d2, np.inf)
    return _mean_of_smallest(d2, k)


def _fixed_order_sum(v):
    """Chunks of CHUNK values summed left to right, then the chunk sums left to right."""
    v = np.asarray(v, np.float64)
    pad = (-len(v)) % CHUNK
    chunks = np.concatenate([v, np.zeros(pad)]).reshape(-1, CHUNK)
    s = np.zeros(len(chunks))
    for j in range(CHUNK):
        s = s + chunks[:, j]                 # + 0.0 on the padding leaves a sum of m >= 0 alone
    total = 0.0
    for c in s.tolist():
        total = total + c
    return total, s


def statistics(m, std_ratio):
    """mu, sigma, threshold and the chunk sums (2, chunks) of the mean distances m."""
    m = np.asarray(m, np.float64)
    n = len(m)
    s1, c1 = _fixed_order_sum(m)
    mu = s1 / n
    d = m - mu
    s2, c2 = _fixed_order_sum(d * d)
    sigma = math.sqrt(s2 / (n - 1))
    return mu, sigma, mu + float(std_ratio) * sigma, np.stack([c1, c2])


def remove_statistical_outliers(xyz, k=20, std_ratio=2.0):
    """-> (keep (N,) bool, m (N,) float64, mu, sigma, threshold)."""
    m = mean_distance(xyz, k)
    mu, sigma, thr, _ = statistics(m, std_ratio)
    return m <= thr, m, mu, sigma, thr
