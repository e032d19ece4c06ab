"""numpy float64 restatement of uniform surface sampling (mesh_sample.py; the casmvs_mesh_sample_*
kernels of csrc/mesh_sample.cu), bit for bit: per-face counts, their offsets and every sample
position.  numpy does not contract a * b + c into an FMA, so each operation below is rounded in
the order written, as the kernels do with __dadd_rn / __dmul_rn.  Never imported by the product."""
from __future__ import annotations

import numpy as np

MAX_ROWS = 65536.0


def counts(verts, faces, spacing):
    """-> (n (F,) int32, count (F,) int64): n = max(1, min(ceil(L / s), 2^16)) with L the
    longest edge in double, count = (n + 1)(n + 2) / 2."""
    p = np.asarray(verts, np.float32).astype(np.float64)[np.asarray(faces, np.int64)]
    a, b, c = p[:, 0], p[:, 1], p[:, 2]

    def length(p, q):
        d = q - p
        return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    L = np.maximum(np.maximum(length(a, b), length(b, c)), length(c, a))
    r = np.minimum(np.ceil(L / np.float64(spacing)), MAX_ROWS)
    n = np.where(r >= 1.0, r, 1.0).astype(np.int64)
    return n.astype(np.int32), (n + 1) * (n + 2) // 2


def offsets(count):
    """Exclusive prefix sum (F,) int64."""
    count = np.asarray(count, np.int64)
    return np.concatenate([[0], np.cumsum(count)[:-1]]).astype(np.int64) if len(count) else \
        np.zeros(0, np.int64)


def row_start(i, n):
    return i * (n + 1) - i * (i - 1) // 2


def decode(k, n):
    """Local index k -> (i, j) of the lattice of a face with n rows, exactly: i is the largest row
    with row_start(i, n) <= k."""
    k, n = np.asarray(k, np.int64), np.asarray(n, np.int64)
    m = (2 * n + 3).astype(np.float64)
    i = ((m - np.sqrt(np.maximum(m * m - 8.0 * k, 0.0))) * 0.5).astype(np.int64)
    i = np.clip(i, 0, n)
    while True:
        down = (i > 0) & (row_start(i, n) > k)
        if not down.any():
            break
        i = i - down
    while True:
        up = (i < n) & (row_start(i + 1, n) <= k)
        if not up.any():
            break
        i = i + up
    return i, k - row_start(i, n)


def sample(verts, faces, spacing):
    """-> (samples (S,3) float32, n, count, offsets) in face-major, then k, order."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    n, cnt = counts(verts, faces, spacing)
    off = offsets(cnt)
    S = int(cnt.sum())
    f = np.repeat(np.arange(len(faces)), cnt)
    k = np.arange(S, dtype=np.int64) - off[f]
    nf = n.astype(np.int64)[f]
    i, j = decode(k, nf)
    u = i.astype(np.float64) / nf.astype(np.float64)
    v = j.astype(np.float64) / nf.astype(np.float64)
    p = np.asarray(verts, np.float32).astype(np.float64)
    a, b, c = p[faces[f, 0]], p[faces[f, 1]], p[faces[f, 2]]
    out = (a + u[:, None] * (b - a)) + v[:, None] * (c - a)
    return out.astype(np.float32), n, cnt, off
