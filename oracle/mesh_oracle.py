"""numpy restatement of csrc/mesh.cu: the TSDF integration in float32 (every operation rounded
to nearest, in the order include/casmvs.h states, so the bits match the kernel) and the
marching-cubes extraction in float64 with the generated case table (casmvsnet_pl_b200/mc_table.py),
with the kernel's vertex and triangle order.  Plus dense analytic signed-distance grids as volumes,
and the mesh topology measures the tests use."""
from __future__ import annotations

import numpy as np

from casmvsnet_pl_b200 import mc_table

BIAS = 1 << 20
f32 = np.float32


def pack_keys(b):
    b = np.asarray(b, dtype=np.int64) + BIAS
    return (b[..., 0] << 42) | (b[..., 1] << 21) | b[..., 2]


def unpack_keys(k):
    k = np.asarray(k, dtype=np.int64)
    return np.stack([(k >> 42) - BIAS, ((k >> 21) & 0x1FFFFF) - BIAS, (k & 0x1FFFFF) - BIAS], -1)


def voxel_indices(keys):
    """(nb*512, 3) int64 voxel index ijk of every voxel, in voxel order."""
    l = np.arange(512)
    local = np.stack([l & 7, (l >> 3) & 7, l >> 6], -1)
    return (unpack_keys(keys)[:, None, :] * 8 + local[None]).reshape(-1, 3)


def brick_keys(points, voxel, trunc):
    """Sorted unique keys of the bricks casmvs_mesh_brick_keys marks for points (N,3) float32,
    and the number of points it drops."""
    p = np.asarray(points, dtype=f32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        lo = np.ceil((p - f32(trunc)) / f32(voxel))
        hi = np.floor((p + f32(trunc)) / f32(voxel))
    ok = ((lo >= -8 * BIAS) & (hi <= 8 * (BIAS - 2) + 7) & (lo <= hi)).all(1)
    blo = lo[ok].astype(np.int64) >> 3
    bhi = np.minimum(hi[ok].astype(np.int64) >> 3, blo + 1)
    ks = [pack_keys(np.minimum(blo + np.array([s & 1, (s >> 1) & 1, s >> 2]), bhi)) for s in range(8)]
    return np.unique(np.concatenate(ks)), int((~ok).sum())


def brick_neighbors(keys):
    keys = np.asarray(keys, dtype=np.int64)
    b = unpack_keys(keys)
    out = np.full((len(keys), 7), -1, dtype=np.int64)
    for o in range(1, 8):
        want = pack_keys(b + np.array([o & 1, (o >> 1) & 1, o >> 2]))
        pos = np.searchsorted(keys, want)
        hit = pos < len(keys)
        hit[hit] = keys[pos[hit]] == want[hit]
        out[hit, o - 1] = pos[hit]
    return out


def integrate(keys, views, voxel, trunc, state=None):
    """views: [(depth (H,W) f32, image (H,W,3) f32, P (4,4) f32)] in order -> (tsdf, weight,
    color (.,3)) float32, continuing from `state` (zeros by default)."""
    ijk = voxel_indices(keys)
    voxel, trunc = f32(voxel), f32(trunc)
    X, Y, Z = (ijk[:, a].astype(f32) * voxel for a in range(3))
    n = len(ijk)
    if state is None:
        s, w, col = np.zeros(n, f32), np.zeros(n, f32), np.zeros((n, 3), f32)
    else:
        s, w, col = (np.array(a, dtype=f32, copy=True) for a in state)
    with np.errstate(all="ignore"):
        for depth, image, P in views:
            P = np.asarray(P, dtype=f32)
            H, W = depth.shape

            def row(r):
                return ((P[r, 0] * X + P[r, 1] * Y) + P[r, 2] * Z) + P[r, 3]
            z, uz, vz = row(2), row(0), row(1)
            fx = np.floor(uz / z + f32(0.5))
            fy = np.floor(vz / z + f32(0.5))
            ok = (z > 0) & (fx >= 0) & (fx < W) & (fy >= 0) & (fy < H)
            px = np.where(ok, fx, 0).astype(np.int64)
            py = np.where(ok, fy, 0).astype(np.int64)
            D = np.asarray(depth, dtype=f32)[py, px]
            ok &= D != 0
            sdf = D - z
            ok &= sdf >= -trunc
            t = np.minimum(f32(1), sdf / trunc)
            w1 = w + f32(1)
            s = np.where(ok, (s * w + t) / w1, s)
            im = np.asarray(image, dtype=f32)[py, px]
            col = np.where(ok[:, None], (col * w[:, None] + im) / w1[:, None], col)
            w = np.where(ok, w1, w)
    return s.astype(f32), w.astype(f32), col.astype(f32)


def _corner_voxels(nbr):
    """(nb*512, 8) voxel index of each cell corner, -1 where unallocated."""
    nb = len(nbr)
    v = np.arange(nb * 512)
    b, l = v >> 9, v & 511
    x, y, z = l & 7, (l >> 3) & 7, l >> 6
    out = np.empty((nb * 512, 8), dtype=np.int64)
    for c in range(8):
        cx, cy, cz = x + (c & 1), y + ((c >> 1) & 1), z + (c >> 2)
        o = (cx >> 3) | ((cy >> 3) << 1) | ((cz >> 3) << 2)
        bb = np.where(o > 0, nbr[b, np.maximum(o - 1, 0)], b)
        out[:, c] = np.where(bb < 0, -1, bb * 512 + ((cz & 7) * 8 + (cy & 7)) * 8 + (cx & 7))
    return out


def extract(keys, tsdf, weight, color, voxel):
    """-> (verts (N,3) f32, colours (N,3) u8, faces (M,3) int32) in the kernel's order."""
    tris, count, mask = mc_table.table()
    nbr = brick_neighbors(keys)
    cv = _corner_voxels(nbr)
    ok = (cv >= 0).all(1)
    ok[ok] = (weight[cv[ok]] > 0).all(1)
    case = np.zeros(len(cv), dtype=np.int64)
    case[ok] = ((tsdf[cv[ok]] < 0) << np.arange(8)).sum(1)
    ntri = np.where(ok, count[case], 0)
    lower = np.array([mc_table.EDGES[e][0] for e in range(12)])
    used = np.zeros(len(cv) * 3, dtype=bool)
    cells = np.nonzero(ntri)[0]
    for e in range(12):
        sel = cells[(mask[case[cells]] >> e) & 1 == 1]
        used[cv[sel, lower[e]] * 3 + e // 4] = True
    vid = np.cumsum(used) - 1
    q = np.nonzero(used)[0]
    v, axis = q // 3, q % 3
    u = cv[v, 1 << axis]
    s0, s1 = tsdf[v].astype(np.float64), tsdf[u].astype(np.float64)
    t = s0 / (s0 - s1)
    ijk = voxel_indices(keys)[v].astype(np.float64)
    ijk[np.arange(len(q)), axis] += t
    verts = (ijk * np.float64(f32(voxel))).astype(f32)
    c0, c1 = color[v].astype(np.float64), color[u].astype(np.float64)
    cols = np.clip(np.rint(c0 + t[:, None] * (c1 - c0)), 0, 255).astype(np.uint8)
    rows, order = [], []
    for k in range(tris.shape[1]):                 # triangle k of every cell that has one
        c = cells[count[case[cells]] > k]
        e = tris[case[c], k].astype(np.int64)      # (n,3) edges
        rows.append(vid[cv[c[:, None], lower[e]] * 3 + e // 4])
        order.append(c * tris.shape[1] + k)
    order = np.concatenate(order)
    faces = np.concatenate(rows)[np.argsort(order, kind="stable")].astype(np.int32)
    return verts, cols, faces.reshape(-1, 3)


def grid_volume(sdf, origin=(0, 0, 0)):
    """A dense grid sdf (X,Y,Z) of voxel values, voxel (0,0,0) at index `origin`, as a volume:
    -> (keys, tsdf, weight, color); voxels of the bricks outside the grid have weight 0."""
    sdf = np.asarray(sdf, dtype=f32)
    o = np.asarray(origin, dtype=np.int64)
    lo, hi = o // 8, (o + np.array(sdf.shape) - 1) // 8
    g = np.stack(np.meshgrid(*[np.arange(a, b + 1) for a, b in zip(lo, hi)], indexing="ij"), -1)
    keys = np.sort(pack_keys(g.reshape(-1, 3)))
    rel = voxel_indices(keys) - o
    inside = ((rel >= 0) & (rel < np.array(sdf.shape))).all(1)
    tsdf = np.zeros(len(rel), f32)
    tsdf[inside] = sdf[tuple(rel[inside].T)]
    weight = inside.astype(f32)
    color = np.zeros((len(rel), 3), f32)
    color[inside] = 128
    return keys, tsdf, weight, color


# ------------------------------------------------------------------------------ mesh measures
def edge_counts(faces):
    """-> (undirected edge -> face count, directed edge -> count) as dicts keyed by tuples."""
    f = np.asarray(faces, dtype=np.int64)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    dk, dc = np.unique(d, axis=0, return_counts=True)
    u = np.sort(d, axis=1)
    uk, uc = np.unique(u, axis=0, return_counts=True)
    return uk, uc, dk, dc


def euler_characteristic(n_verts, faces):
    uk, _, _, _ = edge_counts(faces)
    return int(n_verts) - len(uk) + len(faces)


def is_closed_oriented(faces):
    """Every undirected edge in exactly two faces and every directed edge in exactly one."""
    _, uc, _, dc = edge_counts(faces)
    return bool((uc == 2).all() and (dc == 1).all())


def signed_volume(verts, faces):
    v = np.asarray(verts, dtype=np.float64)[np.asarray(faces)]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)
