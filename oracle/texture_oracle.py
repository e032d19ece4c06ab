"""Numpy restatement of csrc/texture.cu and the textured resolve of csrc/render.cu
(casmvsnet_pl_b200/texture.py, render.render_textured_mesh): the same visibility buffers,
candidate rule, top-K order, smoothing, components, rectangles, packing, atlas bytes and UVs, every
float operation rounded in the kernels' order, so the GPU results must match bit for bit.  Test
infrastructure only.

    out = texture_mesh(verts, colours, faces, images, Ps)      # dict of every stage
    image, depth = render_textured_mesh(verts, faces, uv, page, atlas, P, (W, H))
"""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from oracle import render_oracle as R

K, PAD, MIN_COS, DEPTH_SCALE = 4, 2, 0.1, np.float32(1.01)
SMOOTH_ROUNDS, PAGE_SIDE, MAX_PAGE_SIDE, FLAT = 4, 4096, 16384, 4
f32 = np.float32


def eye_of(P):
    P = np.asarray(P, np.float32).astype(np.float64)
    return -np.linalg.solve(P[:3, :3], P[:3, 3])


def neighbours(faces):
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    F = len(f)
    nbr = np.full(3 * F, -1, np.int32)
    if F == 0:
        return nbr.reshape(0, 3)
    g = np.roll(f, -1, 1)
    key = ((np.minimum(f, g) << 32) | np.maximum(f, g)).reshape(-1)
    _, inv, cnt = np.unique(key, return_inverse=True, return_counts=True)
    order = np.argsort(inv, kind="stable")
    start = np.cumsum(cnt) - cnt
    two = np.nonzero(cnt == 2)[0]
    c0, c1 = order[start[two]], order[start[two] + 1]
    ok = c0 // 3 != c1 // 3
    c0, c1 = c0[ok], c1[ok]
    nbr[c0], nbr[c1] = c1 // 3, c0 // 3
    return nbr.reshape(F, 3)


def key_buffer(verts, faces, P, wh):
    """The view's visibility buffer: render_oracle's raster pass."""
    nv = len(np.asarray(verts).reshape(-1, 3))
    return R.render_mesh(verts, np.zeros((nv, 3), np.uint8), faces, P, np.zeros(3, np.float32), wh)[2]


def _dot(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def view_candidates(verts, faces, P, wh, zbuf):
    """-> (candidate mask (F,), score (F,) float32) of one view."""
    W, H = wh
    x = np.asarray(verts, np.float32).reshape(-1, 3)[np.asarray(faces, np.int64).reshape(-1, 3)]
    xd = x.astype(np.float64)
    e1, e2 = xd[:, 1] - xd[:, 0], xd[:, 2] - xd[:, 0]
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1],
                  e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    nn = _dot(n, n)
    cd = ((xd[:, 0] + xd[:, 1]) + xd[:, 2]) / 3.0
    cf = ((x[:, 0] + x[:, 1]) + x[:, 2]) / f32(3)
    F = len(x)
    pts = np.concatenate([x[:, 0], x[:, 1], x[:, 2], cf])
    u, v, w, ok = R.project(P, pts)
    u, v, w, ok = (a.reshape(4, F) for a in (u, v, w, ok))
    m = (nn > 0) & ok.all(0)
    with np.errstate(all="ignore"):
        for k in range(3):
            m &= (u[k] >= PAD) & (u[k] <= W - 1 - PAD) & (v[k] >= PAD) & (v[k] <= H - 1 - PAD)
        d = cd - eye_of(P)
        m &= np.abs(_dot(n, d)) >= MIN_COS * (np.sqrt(nn) * np.sqrt(_dot(d, d)))
    idx = np.nonzero(m)[0]
    for k in range(4):
        px = np.rint(u[k, idx]).astype(np.int64)
        py = np.rint(v[k, idx]).astype(np.int64)
        key = zbuf[py * W + px]
        dep = (key >> np.uint64(32)).astype(np.uint32).view(np.float32)
        good = (key != R.EMPTY) & (w[k, idx] <= dep * DEPTH_SCALE)
        m[idx[~good]] = False
        idx = idx[good]
    ud, vd = u.astype(np.float64), v.astype(np.float64)
    a = (ud[1] - ud[0]) * (vd[2] - vd[0]) - (vd[1] - vd[0]) * (ud[2] - ud[0])
    return m, (0.5 * np.abs(a)).astype(np.float32)


def candidates(verts, faces, Ps, whs, zbufs):
    F = len(np.asarray(faces).reshape(-1, 3))
    sc = np.zeros((F, K), np.float32)
    vw = np.full((F, K), -1, np.int32)
    rows = np.arange(F)
    for vi, (P, wh, zb) in enumerate(zip(Ps, whs, zbufs)):
        m, s = view_candidates(verts, faces, P, wh, zb)
        better = (vw < 0) | (s[:, None] > sc)
        pos = np.where(better.any(1), better.argmax(1), K)
        ins = m & (pos < K)
        for j in range(K - 1, 0, -1):
            sh = ins & (j > pos)
            sc[sh, j], vw[sh, j] = sc[sh, j - 1], vw[sh, j - 1]
        r = rows[ins]
        sc[r, pos[ins]], vw[r, pos[ins]] = s[ins], vi
    return sc, vw


def smooth_round(nbr, sc, vw, lin):
    l = np.where(nbr >= 0, lin[np.maximum(nbr, 0)], -1)
    L = np.where((l[:, 0] >= 0) & ((l[:, 0] == l[:, 1]) | (l[:, 0] == l[:, 2])), l[:, 0],
                 np.where((l[:, 1] >= 0) & (l[:, 1] == l[:, 2]), l[:, 1], -1))
    thr = f32(0.5) * sc[:, 0]
    take = (L >= 0) & ((vw == L[:, None]) & (sc >= thr[:, None])).any(1)
    return np.where(take, L, lin).astype(np.int32)


def smooth(nbr, sc, vw, labels, rounds=SMOOTH_ROUNDS):
    for _ in range(rounds):
        labels = smooth_round(nbr, sc, vw, labels)
    return labels


def components(nbr, labels):
    F = len(labels)
    f = np.repeat(np.arange(F), 3)
    g = nbr.reshape(-1).astype(np.int64)
    e = (g >= 0) & (labels[f] >= 0) & (labels[f] == labels[np.maximum(g, 0)])
    A = coo_matrix((np.ones(int(e.sum())), (f[e], g[e])), shape=(F, F))
    _, lab = connected_components(A, directed=False)
    root = np.full(lab.max() + 1 if F else 0, F, np.int64)
    np.minimum.at(root, lab, np.arange(F))
    return root[lab].astype(np.int32)


def rects(verts, faces, labels, comp, Ps):
    F = len(labels)
    rect = np.tile(np.array([2**31 - 1, 2**31 - 1, -2**31, -2**31], np.int64), (F, 1))
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    x = np.asarray(verts, np.float32).reshape(-1, 3)
    for vi in np.unique(labels[labels >= 0]):
        idx = np.nonzero(labels == vi)[0]
        u, v, _, _ = R.project(Ps[vi], x[f[idx]].reshape(-1, 3))
        u, v = u.reshape(-1, 3), v.reshape(-1, 3)
        c = comp[idx]
        np.minimum.at(rect[:, 0], c, np.floor(u.min(1)).astype(np.int64) - PAD)
        np.minimum.at(rect[:, 1], c, np.floor(v.min(1)).astype(np.int64) - PAD)
        np.maximum.at(rect[:, 2], c, np.ceil(u.max(1)).astype(np.int64) + PAD)
        np.maximum.at(rect[:, 3], c, np.ceil(v.max(1)).astype(np.int64) + PAD)
    return rect.astype(np.int32)


def pack(ids, w, h, S):
    order = np.lexsort((np.asarray(ids), -np.asarray(w, np.int64), -np.asarray(h, np.int64)))
    page, ox, oy = (np.zeros(len(ids), np.int32) for _ in range(3))
    p = x = y = shelf = 0
    for i in order:
        if x + w[i] > S:
            x, y, shelf = 0, y + shelf, 0
        if y + h[i] > S:
            p, x, y, shelf = p + 1, 0, 0, 0
        page[i], ox[i], oy[i] = p, x, y
        x += int(w[i])
        shelf = max(shelf, int(h[i]))
    return page, ox, oy, (p + 1 if len(ids) else 0)


def texture_mesh(verts, colours, faces, images, Ps, rounds=SMOOTH_ROUNDS, zbufs=None):
    """-> dict: score, view, nbr, labels0, labels, comp0, comp, rect, charts, S, uv, page, atlas."""
    verts = np.asarray(verts, np.float32).reshape(-1, 3)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    colours = np.asarray(colours, np.uint8).reshape(-1, 3)
    Ps = [np.asarray(P, np.float32) for P in Ps]
    whs = [(im.shape[1], im.shape[0]) for im in images]
    if zbufs is None:
        zbufs = [key_buffer(verts, faces, P, wh) for P, wh in zip(Ps, whs)]
    sc, vw = candidates(verts, faces, Ps, whs, zbufs)
    nbr = neighbours(faces)
    labels0 = vw[:, 0].copy()
    labels = smooth(nbr, sc, vw, labels0, rounds)
    comp0, comp = components(nbr, labels0), components(nbr, labels)
    rect = rects(verts, faces, labels, comp, Ps)
    F = len(faces)
    roots = np.nonzero(comp == np.arange(F))[0]
    lab = labels[roots]
    box = np.where((lab < 0)[:, None], np.array([0, 0, FLAT - 1, FLAT - 1]), rect[roots])
    w, h = box[:, 2] - box[:, 0] + 1, box[:, 3] - box[:, 1] + 1
    side = int(max(w.max(initial=0), h.max(initial=0)))
    assert side <= MAX_PAGE_SIDE
    S = PAGE_SIDE
    while S < side:
        S *= 2
    page_c, ox, oy, n_pages = pack(roots, w, h, S)
    charts = np.concatenate([roots[:, None], lab[:, None], box, page_c[:, None], ox[:, None],
                             oy[:, None]], 1).astype(np.int32)
    atlas = np.zeros((n_pages, S, S, 3), np.uint8)
    for c in charts:
        r, vi, x0, y0, x1, y1, pg, cx, cy = (int(a) for a in c)
        if vi < 0:
            atlas[pg, cy:cy + FLAT, cx:cx + FLAT] = (colours[faces[r]].astype(np.int64).sum(0) + 1) // 3
        else:
            atlas[pg, cy:cy + y1 - y0 + 1, cx:cx + x1 - x0 + 1] = images[vi][y0:y1 + 1, x0:x1 + 1]
    slot = np.searchsorted(roots, comp)
    ch = charts[slot].astype(np.float64)
    uv = np.zeros((F, 3, 2), np.float32)
    flat = labels < 0
    for k, (cx, cy) in enumerate(((1.5, 1.5), (2.5, 1.5), (1.5, 2.5))):
        uv[flat, k, 0] = ((ch[flat, 7] + cx) / S).astype(np.float32)
        uv[flat, k, 1] = (1.0 - (ch[flat, 8] + cy) / S).astype(np.float32)
    for vi in np.unique(labels[~flat]):
        idx = np.nonzero(labels == vi)[0]
        u, v, _, _ = R.project(Ps[vi], verts[faces[idx]].reshape(-1, 3))
        u, v = u.reshape(-1, 3).astype(np.float64), v.reshape(-1, 3).astype(np.float64)
        c = ch[idx]
        uv[idx, :, 0] = ((((u - c[:, 2:3]) + c[:, 7:8]) + 0.5) / S).astype(np.float32)
        uv[idx, :, 1] = (1.0 - (((v - c[:, 3:4]) + c[:, 8:9]) + 0.5) / S).astype(np.float32)
    return dict(score=sc, view=vw, nbr=nbr, labels0=labels0, labels=labels, comp0=comp0, comp=comp,
                rect=rect, charts=charts, S=S, uv=uv, page=charts[slot, 6].astype(np.int32),
                atlas=atlas, zbufs=zbufs)


def render_textured_mesh(verts, faces, uv, page, atlas, P, wh):
    """-> (image (H,W,3) uint8, depth (H,W) float32): the raster pass, then the winner's UV
    interpolated perspective-correctly and the page sampled bilinearly (texel centres at i + 0.5,
    indices clamped), unshaded."""
    W, H = wh
    verts = np.asarray(verts, np.float32).reshape(-1, 3)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    uv = np.asarray(uv, np.float32).reshape(-1, 3, 2)
    atlas = np.asarray(atlas, np.uint8)
    S = atlas.shape[1]
    zbuf = key_buffer(verts, faces, P, wh)
    U, V, Wd, _, _ = R._setup(verts, faces, P, wh)
    image = np.broadcast_to(R.BACKGROUND, (W * H, 3)).copy()
    depth = np.zeros(W * H, np.float32)
    pix = np.nonzero(zbuf != R.EMPTY)[0]
    t = (zbuf[pix] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    depth[pix] = (zbuf[pix] >> np.uint64(32)).astype(np.uint32).view(np.float32)
    _, q, den, _ = R.tri_depth(U[t], V[t], Wd[t], (pix % W).astype(np.float32),
                               (pix // W).astype(np.float32))
    Sf = f32(S)
    with np.errstate(all="ignore"):
        c = uv[t]
        tu = ((q[:, 0] * c[:, 0, 0] + q[:, 1] * c[:, 1, 0]) + q[:, 2] * c[:, 2, 0]) / den
        tv = ((q[:, 0] * c[:, 0, 1] + q[:, 1] * c[:, 1, 1]) + q[:, 2] * c[:, 2, 1]) / den
        x = np.fmin(np.fmax(tu * Sf - f32(0.5), f32(-1)), Sf)
        y = np.fmin(np.fmax((f32(1) - tv) * Sf - f32(0.5), f32(-1)), Sf)
    fx, fy = np.floor(x), np.floor(y)
    ax, ay = x - fx, y - fy
    ix, iy = fx.astype(np.int64), fy.astype(np.int64)
    x0, x1 = np.clip(ix, 0, S - 1), np.clip(ix + 1, 0, S - 1)
    y0, y1 = np.clip(iy, 0, S - 1), np.clip(iy + 1, 0, S - 1)
    pg = np.asarray(page, np.int64)[t]
    for ch in range(3):
        c00 = atlas[pg, y0, x0, ch].astype(np.float32)
        c10 = atlas[pg, y0, x1, ch].astype(np.float32)
        c01 = atlas[pg, y1, x0, ch].astype(np.float32)
        c11 = atlas[pg, y1, x1, ch].astype(np.float32)
        r0 = (f32(1) - ax) * c00 + ax * c10
        r1 = (f32(1) - ax) * c01 + ax * c11
        val = np.floor(((f32(1) - ay) * r0 + ay * r1) + f32(0.5))
        image[pix, ch] = np.fmin(f32(255), np.fmax(f32(0), val)).astype(np.uint8)
    return image.reshape(H, W, 3), depth.reshape(H, W)
