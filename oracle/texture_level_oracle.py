"""Numpy restatement of csrc/texture_level.cu (texture.py's seam levelling): the unknowns, the
seam records and pairs, the seam colours, the CSR system and its right-hand side, the texel owners
and the applied atlas, every double operation in the kernels' order, so the GPU results must match
bit for bit.  The solve is direct (scipy's sparse LU on the same matrix) where the GPU runs
conjugate gradients.  Test infrastructure only.

    out = level(verts, faces, labels, slot, charts, Ps, images, nbr, atlas)   # dict of every step
"""
import numpy as np
from scipy.sparse import csc_matrix, csr_matrix
from scipy.sparse.linalg import splu

from oracle import render_oracle as R

SEAM_SAMPLES, SMOOTH_WEIGHT, EPS, REACH = 8, 10.0, 1e-4, 1.5
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
LO32 = np.int64(0xFFFFFFFF)


def unknowns(faces, labels, slot):
    """-> (keys (n,) int64 ascending = (slot << 32) | vertex, corner (F,3) int32, -1 when flat)."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    keys = (np.asarray(slot, np.int64)[:, None] << 32) | faces
    keys = np.where((np.asarray(labels) >= 0)[:, None], keys, -1)
    unk = np.unique(keys[keys >= 0])
    corner = np.where(keys >= 0, np.searchsorted(unk, keys), -1).astype(np.int32)
    return unk, corner


def _pair(a, b):
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    return (np.minimum(a, b) << 32) | np.maximum(a, b)


def edges(nbr, faces, labels, slot, corner):
    """-> (rec_key, rec_sub) of the seam endpoint records sorted by (key, record), the distinct
    smoothing-edge keys."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    nbr = np.asarray(nbr, np.int64).reshape(-1, 3)
    labels, slot = np.asarray(labels), np.asarray(slot)
    F = len(faces)
    view = labels >= 0
    k1 = np.array([1, 2, 0])
    a, b = corner.astype(np.int64), corner[:, k1].astype(np.int64)
    sm = view[:, None] & (a != b)
    smooth = np.unique(_pair(a, b)[sm])
    g = np.maximum(nbr, 0)
    f = np.arange(F)[:, None]
    seam = ((nbr >= 0) & (f < nbr) & view[:, None] & (labels[g] >= 0) & (slot[:, None] != slot[g]))
    rec_key = np.full((F, 3, 2), -1, np.int64)
    for e in range(2):
        kk = np.arange(3) if e == 0 else k1
        vtx = faces[:, kk]                                            # (F,3)
        other = np.full((F, 3), -1, np.int64)
        for j in (2, 1, 0):                                          # the first match wins
            other = np.where(faces[g, j] == vtx, corner[g, j], other)
        rec_key[:, :, e] = np.where(seam, _pair(corner[np.arange(F)[:, None], kk], other), -1)
    rec_key = rec_key.reshape(-1)
    sub = np.nonzero(rec_key >= 0)[0]
    order = np.argsort(rec_key[sub], kind="stable")
    return rec_key[sub][order], sub[order].astype(np.int64), smooth


def _bilinear(img, u, v):
    H, W = img.shape[:2]
    u = np.fmin(np.fmax(u, 0.0), float(W - 1))
    v = np.fmin(np.fmax(v, 0.0), float(H - 1))
    fx, fy = np.floor(u), np.floor(v)
    ax, ay = u - fx, v - fy
    x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    im = img.astype(np.float64)
    c00, c10, c01, c11 = im[y0, x0], im[y0, x1], im[y1, x0], im[y1, x1]
    ax, ay = ax[:, None], ay[:, None]
    r0 = (1.0 - ax) * c00 + ax * c10
    r1 = (1.0 - ax) * c01 + ax * c11
    return (1.0 - ay) * r0 + ay * r1


def _row(P, X, Y, Z):
    return ((P[:, 0] * X + P[:, 1] * Y) + P[:, 2] * Z) + P[:, 3]


def samples(verts, faces, labels, slot, nbr, rec_sub, Ps, images):
    """-> rec (R,6): the (1 - t)-weighted sums of the samples in the lower chart's view (0..2)
    and the upper chart's (3..5)."""
    verts = np.asarray(verts, np.float32).reshape(-1, 3).astype(np.float64)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    nbr = np.asarray(nbr, np.int64).reshape(-1)
    labels, slot = np.asarray(labels), np.asarray(slot)
    c, e = rec_sub >> 1, rec_sub & 1
    f, k = c // 3, c % 3
    k1 = np.where(k == 2, 0, k + 1)
    g = nbr[c]
    low = slot[f] < slot[g]
    va, vb = labels[np.where(low, f, g)], labels[np.where(low, g, f)]
    x0 = verts[faces[f, np.where(e == 1, k1, k)]]
    x1 = verts[faces[f, np.where(e == 1, k, k1)]]
    P64 = np.stack([np.asarray(P, np.float32).astype(np.float64) for P in Ps]) if len(Ps) else None
    rec = np.zeros((len(rec_sub), 6))
    for s in range(SEAM_SAMPLES):
        t = s / SEAM_SAMPLES
        wt = 1.0 - t
        X = x0 + t * (x1 - x0)
        for col, vw in ((0, va), (3, vb)):
            P = P64[vw]
            w = _row(P[:, 2], X[:, 0], X[:, 1], X[:, 2])
            u = _row(P[:, 0], X[:, 0], X[:, 1], X[:, 2]) / w
            v = _row(P[:, 1], X[:, 0], X[:, 1], X[:, 2]) / w
            val = np.zeros((len(rec_sub), 3))
            for i in np.unique(vw):
                m = vw == i
                val[m] = _bilinear(np.asarray(images[i]), u[m], v[m])
            rec[:, col:col + 3] = rec[:, col:col + 3] + wt * val
    return rec


def pairs(rec_key, rec):
    """-> (pair keys (P,) ascending, fpair (P,6): f_a, f_b)."""
    keys, idx = np.unique(rec_key, return_inverse=True)
    wrec = 0.0
    for s in range(SEAM_SAMPLES):
        wrec = wrec + (1.0 - s / SEAM_SAMPLES)
    num = np.zeros((len(keys), 6))
    den = np.zeros(len(keys))
    np.add.at(num, idx, rec)                                        # in record order
    np.add.at(den, idx, np.full(len(idx), wrec))
    return keys, num / den[:, None]


def system(pair_keys, smooth_keys, n, fpair):
    """-> (rowptr (n+1), col (nnz) int32, val (nnz), diag (n), rhs (n,3))."""
    lo_p, hi_p = pair_keys >> 32, pair_keys & LO32
    lo_s, hi_s = smooth_keys >> 32, smooth_keys & LO32
    a = np.arange(n, dtype=np.int64)
    ekey = np.concatenate([(lo_p << 32) | hi_p, (hi_p << 32) | lo_p, (lo_s << 32) | hi_s,
                           (hi_s << 32) | lo_s, (a << 32) | a])
    etype = np.concatenate([np.arange(len(pair_keys)), np.arange(len(pair_keys)),
                            np.full(2 * len(smooth_keys), -2), np.full(n, -1)]).astype(np.int64)
    order = np.argsort(ekey)
    ekey, etype = ekey[order], etype[order]
    row, col = ekey >> 32, (ekey & LO32)
    rowptr = np.searchsorted(row, np.arange(n + 1)).astype(np.int32)
    off = etype != -1
    val = np.where(etype == -2, -SMOOTH_WEIGHT, -1.0)
    s = np.zeros(n)
    np.add.at(s, row[off], val[off])
    diag = -s + EPS
    val[~off] = diag[row[~off]]
    seam = etype >= 0
    fp = fpair[etype[seam]]
    low = (row[seam] < col[seam])[:, None]
    contrib = np.where(low, fp[:, 3:] - fp[:, :3], fp[:, :3] - fp[:, 3:])
    rhs = np.zeros((n, 3))
    np.add.at(rhs, row[seam], contrib)
    return rowptr, col.astype(np.int32), val, diag, rhs


def solve(rowptr, col, val, rhs):
    """The direct solution of A g = rhs, (n,3)."""
    n = len(rowptr) - 1
    if n == 0:
        return np.zeros((0, 3))
    A = csc_matrix(csr_matrix((val, col, rowptr), shape=(n, n)))
    return splu(A).solve(np.ascontiguousarray(rhs))


def nearest(u, v, px, py):
    """Point-to-triangle in 2D, vectorised: u, v (M,3) float64, px, py (M,) -> (dist (M,),
    l (M,3) barycentrics of the nearest point)."""
    M = len(px)
    with np.errstate(all="ignore"):
        area = (u[:, 1] - u[:, 0]) * (v[:, 2] - v[:, 0]) - (v[:, 1] - v[:, 0]) * (u[:, 2] - u[:, 0])
        li = []
        for k in range(3):
            a, b = (k + 1) % 3, (k + 2) % 3
            li.append(((u[:, a] - px) * (v[:, b] - py) - (v[:, a] - py) * (u[:, b] - px)) / area)
        inside = (area != 0) & (li[0] >= 0) & (li[1] >= 0) & (li[2] >= 0)
        best = np.full(M, np.inf)
        bt = np.zeros(M)
        bk = np.zeros(M, np.int64)
        for k in range(3):
            k1 = (k + 1) % 3
            dx, dy = u[:, k1] - u[:, k], v[:, k1] - v[:, k]
            d2e = dx * dx + dy * dy
            t = np.where(d2e > 0, ((px - u[:, k]) * dx + (py - v[:, k]) * dy) / d2e, 0.0)
            t = np.fmin(np.fmax(t, 0.0), 1.0)
            ex, ey = px - (u[:, k] + t * dx), py - (v[:, k] + t * dy)
            d2 = ex * ex + ey * ey
            upd = d2 < best
            best, bt, bk = np.where(upd, d2, best), np.where(upd, t, bt), np.where(upd, k, bk)
    l = np.zeros((M, 3))
    rows = np.arange(M)
    l[rows, bk] = 1.0 - bt
    l[rows, (bk + 1) % 3] = bt
    l = np.where(inside[:, None], np.stack(li, 1), l)
    return np.where(inside, 0.0, np.sqrt(best)), l


def face_uv(verts, faces, labels, Ps, idx):
    """The float32 projections (texture.uvs') of faces idx in their label's view, as float64."""
    verts = np.asarray(verts, np.float32).reshape(-1, 3)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    u, v = np.zeros((len(idx), 3)), np.zeros((len(idx), 3))
    lab = labels[idx]
    for L in np.unique(lab):
        m = lab == L
        uu, vv, _, _ = R.project(np.asarray(Ps[L], np.float32), verts[faces[idx[m]]].reshape(-1, 3))
        u[m], v[m] = uu.reshape(-1, 3), vv.reshape(-1, 3)
    return u, v


def owners(verts, faces, labels, slot, charts, Ps, S, n_pages):
    """-> owner (pages,S,S) uint64: (f32 distance bits << 32) | face, least per texel; ~0 free."""
    labels, slot = np.asarray(labels), np.asarray(slot)
    owner = np.full(n_pages * S * S, EMPTY, np.uint64)
    idx = np.nonzero(labels >= 0)[0]
    if not len(idx):
        return owner.reshape(n_pages, S, S)
    u, v = face_uv(verts, faces, labels, Ps, idx)
    c = charts[slot[idx]].astype(np.int64)
    xlo = np.maximum(c[:, 2], np.ceil(u.min(1) - REACH).astype(np.int64))
    xhi = np.minimum(c[:, 4], np.floor(u.max(1) + REACH).astype(np.int64))
    ylo = np.maximum(c[:, 3], np.ceil(v.min(1) - REACH).astype(np.int64))
    yhi = np.minimum(c[:, 5], np.floor(v.max(1) + REACH).astype(np.int64))
    nx, ny = np.maximum(xhi - xlo + 1, 0), np.maximum(yhi - ylo + 1, 0)
    cnt = nx * ny
    j = np.repeat(np.arange(len(idx)), cnt)
    i = np.arange(len(j)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    x, y = xlo[j] + i % nx[j], ylo[j] + i // nx[j]
    dist, _ = nearest(u[j], v[j], x.astype(np.float64), y.astype(np.float64))
    ok = dist <= REACH
    j, x, y, dist = j[ok], x[ok], y[ok], dist[ok]
    key = (dist.astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | \
        idx[j].astype(np.uint64)
    cj = c[j]
    t = cj[:, 6] * S * S + (cj[:, 8] + y - cj[:, 3]) * S + (cj[:, 7] + x - cj[:, 2])
    np.minimum.at(owner, t, key)
    return owner.reshape(n_pages, S, S)


def apply(owner, verts, faces, labels, slot, charts, Ps, corner, g, atlas):
    """-> the atlas with every owned texel offset by its owner's interpolated g."""
    labels, slot = np.asarray(labels), np.asarray(slot)
    atlas = np.array(atlas, np.uint8)
    S = atlas.shape[1]
    flat = owner.reshape(-1)
    t = np.nonzero(flat != EMPTY)[0]
    f = (flat[t] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    rem = t % (S * S)
    ty, tx = rem // S, rem % S
    c = charts[slot[f]].astype(np.int64)
    u, v = face_uv(verts, faces, labels, Ps, f)
    _, l = nearest(u, v, (c[:, 2] + tx - c[:, 7]).astype(np.float64),
                   (c[:, 3] + ty - c[:, 8]).astype(np.float64))
    cu = corner[f].astype(np.int64)
    off = (l[:, 0:1] * g[cu[:, 0]] + l[:, 1:2] * g[cu[:, 1]]) + l[:, 2:3] * g[cu[:, 2]]
    A = atlas.reshape(-1, 3)
    A[t] = np.fmin(np.fmax(np.rint(A[t].astype(np.float64) + off), 0.0), 255.0).astype(np.uint8)
    return atlas


def seam_rms(fpair, g=None, pair_keys=None):
    """RMS over pairs and channels of f_a - f_b, or of f_a + g_a - f_b - g_b."""
    if not len(fpair):
        return 0.0
    d = fpair[:, :3] - fpair[:, 3:]
    if g is not None:
        d = d + g[pair_keys >> 32] - g[pair_keys & LO32]
    return float(np.sqrt(np.mean(d * d)))


def level(verts, faces, labels, slot, charts, Ps, images, nbr, atlas, g=None):
    """Every step; g (n,3) replaces the direct solution in the owners / apply steps when given."""
    labels, slot = np.asarray(labels), np.asarray(slot)
    charts = np.asarray(charts)
    unk, corner = unknowns(faces, labels, slot)
    rec_key, rec_sub, smooth = edges(nbr, faces, labels, slot, corner)
    rec = samples(verts, faces, labels, slot, nbr, rec_sub, Ps, images)
    pair_keys, fpair = pairs(rec_key, rec)
    rowptr, col, val, diag, rhs = system(pair_keys, smooth, len(unk), fpair)
    g_direct = solve(rowptr, col, val, rhs)
    gg = g_direct if g is None else g
    atlas = np.asarray(atlas)
    own = owners(verts, faces, labels, slot, charts, Ps, atlas.shape[1], len(atlas))
    out = apply(own, verts, faces, labels, slot, charts, Ps, corner, gg, atlas)
    return dict(unknowns=unk, corner=corner, rec_key=rec_key, rec_sub=rec_sub, smooth=smooth,
                rec=rec, pair_keys=pair_keys, fpair=fpair, rowptr=rowptr, col=col, val=val,
                diag=diag, rhs=rhs, g=g_direct, owner=own, atlas=out,
                seam_rms_before=seam_rms(fpair), seam_rms_after=seam_rms(fpair, gg, pair_keys))
