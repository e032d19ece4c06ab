"""Numpy float32 restatement of csrc/render.cu (casmvsnet_pl_b200/render.py): the same
projection, key, tie rule, coverage, interpolation and shade, with every operation rounded to
float32 in the kernels' order, so the GPU images and depth maps must match bit for bit.  Test
infrastructure only.

    image, depth = render_points(xyz, rgb, P, (W, H), point_size)
    image, depth = render_mesh(verts, colours, faces, P, eye, (W, H))
"""
import numpy as np

EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
BACKGROUND = np.array([128, 128, 255], np.uint8)
SMALL_BOX = 8
_CHUNK = 1 << 22                  # (face, pixel) pairs per rasterisation step
f32 = np.float32


def _row(A, X, Y, Z):
    return ((A[0] * X + A[1] * Y) + A[2] * Z) + A[3]


def project(P, xyz):
    """-> u, v, w (float32) and ok: finite X, Y, Z, w, u, v and w > 0."""
    P = np.asarray(P, np.float32).reshape(4, 4)
    X, Y, Z = (np.ascontiguousarray(xyz[:, a], np.float32) for a in range(3))
    with np.errstate(all="ignore"):
        ok = np.isfinite(X) & np.isfinite(Y) & np.isfinite(Z)
        w = _row(P[2], X, Y, Z)
        ok &= (w > 0) & np.isfinite(w)
        u = _row(P[0], X, Y, Z) / w
        v = _row(P[1], X, Y, Z) / w
        ok &= np.isfinite(u) & np.isfinite(v)
    return u, v, w, ok


def keys(w, idx):
    return (w.astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | \
        idx.astype(np.uint64)


def render_points(xyz, rgb, P, wh, point_size=1):
    """-> (image (H,W,3) uint8, depth (H,W) float32, zbuf (H*W,) uint64)."""
    W, H = wh
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    u, v, w, ok = project(P, xyz)
    h = f32(0.5 * point_size)
    with np.errstate(all="ignore"):
        x0, x1 = np.ceil(u - h), np.ceil(u + h) - f32(1)
        y0, y1 = np.ceil(v - h), np.ceil(v + h) - f32(1)
        ok &= ~((x1 < 0) | (y1 < 0) | (x0 > W - 1) | (y0 > H - 1))
    idx = np.nonzero(ok)[0]
    xa = np.maximum(x0[idx], 0).astype(np.int64)
    xb = np.minimum(x1[idx], W - 1).astype(np.int64)
    ya = np.maximum(y0[idx], 0).astype(np.int64)
    yb = np.minimum(y1[idx], H - 1).astype(np.int64)
    k = keys(w[idx], idx)
    zbuf = np.full(W * H, EMPTY, np.uint64)
    for dy in range(point_size + 1):
        for dx in range(point_size + 1):
            m = (xa + dx <= xb) & (ya + dy <= yb)
            np.minimum.at(zbuf, (ya[m] + dy) * W + xa[m] + dx, k[m])
    drawn = zbuf != EMPTY
    image = np.broadcast_to(BACKGROUND, (W * H, 3)).copy()
    depth = np.zeros(W * H, np.float32)
    win = (zbuf[drawn] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    image[drawn] = np.asarray(rgb, np.uint8).reshape(-1, 3)[win]
    depth[drawn] = (zbuf[drawn] >> np.uint64(32)).astype(np.uint32).view(np.float32)
    return image.reshape(H, W, 3), depth.reshape(H, W), zbuf


def edge(ax, ay, bx, by, px, py):
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax)


def _setup(verts, faces, P, wh):
    """Per face: projected corners (3 arrays each of shape (M,3)), drawn mask, clamped box."""
    W, H = wh
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(faces) and (faces.min() < 0 or faces.max() >= len(verts)):
        raise ValueError("a face index lies outside [0, n_vertices)")
    u, v, w, ok = project(P, np.asarray(verts, np.float32).reshape(-1, 3))
    U, V, Wd = u[faces], v[faces], w[faces]
    drawn = ok[faces].all(1)
    with np.errstate(all="ignore"):
        area = edge(U[:, 0], V[:, 0], U[:, 1], V[:, 1], U[:, 2], V[:, 2])
        drawn &= (area != 0) & np.isfinite(area)
        lx = np.ceil(np.minimum(np.minimum(U[:, 0], U[:, 1]), U[:, 2]))
        hx = np.floor(np.maximum(np.maximum(U[:, 0], U[:, 1]), U[:, 2]))
        ly = np.ceil(np.minimum(np.minimum(V[:, 0], V[:, 1]), V[:, 2]))
        hy = np.floor(np.maximum(np.maximum(V[:, 0], V[:, 1]), V[:, 2]))
        drawn &= ~((hx < 0) | (hy < 0) | (lx > W - 1) | (ly > H - 1) | (lx > hx) | (ly > hy))
        box = [np.where(drawn, np.clip(b, 0, m), 0).astype(np.int64)
               for b, m in ((lx, W - 1), (hx, W - 1), (ly, H - 1), (hy, H - 1))]
    return U, V, Wd, drawn, box


def tri_depth(U, V, Wd, px, py):
    """Coverage and perspective-correct depth at pixel centres (px, py) float32 of the faces
    U, V, Wd (n,3) -> covered, q (n,3), den, w."""
    with np.errstate(all="ignore"):
        e0 = edge(U[:, 1], V[:, 1], U[:, 2], V[:, 2], px, py)
        e1 = edge(U[:, 2], V[:, 2], U[:, 0], V[:, 0], px, py)
        e2 = edge(U[:, 0], V[:, 0], U[:, 1], V[:, 1], px, py)
        cov = ((e0 >= 0) & (e1 >= 0) & (e2 >= 0)) | ((e0 <= 0) & (e1 <= 0) & (e2 <= 0))
        q = np.stack([e0 / Wd[:, 0], e1 / Wd[:, 1], e2 / Wd[:, 2]], 1)
        den = (q[:, 0] + q[:, 1]) + q[:, 2]
        w = ((e0 + e1) + e2) / den
        cov &= (w > 0) & np.isfinite(w)
    return cov, q, den, w


def face_shade(a, b, c, eye):
    """0.3 + 0.7 min(1, |n.d| / (|n| |d|)) per face (float32), 0.3 when the divisor is 0."""
    eye = np.asarray(eye, np.float32)
    e1, e2 = b - a, c - a
    d = ((a + b) + c) / f32(3) - eye
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1],
                  e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)

    def dot(x, y):
        return (x[:, 0] * y[:, 0] + x[:, 1] * y[:, 1]) + x[:, 2] * y[:, 2]
    with np.errstate(all="ignore"):
        den = np.sqrt(dot(n, n)) * np.sqrt(dot(d, d))
        cs = np.abs(dot(n, d)) / den
        cs = np.where((den > 0) & np.isfinite(cs), np.minimum(cs, f32(1)), f32(0)).astype(np.float32)
    return f32(0.3) + f32(0.7) * cs


def render_mesh(verts, colours, faces, P, eye, wh):
    """-> (image (H,W,3) uint8, depth (H,W) float32, zbuf (H*W,) uint64); eye is the camera
    centre (float32, render.camera_centre)."""
    W, H = wh
    verts = np.asarray(verts, np.float32).reshape(-1, 3)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    U, V, Wd, drawn, (x0, x1, y0, y1) = _setup(verts, faces, P, wh)
    zbuf = np.full(W * H, EMPTY, np.uint64)
    ids = np.nonzero(drawn)[0]
    bw, bh = (x1 - x0 + 1)[ids], (y1 - y0 + 1)[ids]
    npx = bw * bh
    ends = np.cumsum(npx)
    s = 0
    while s < len(ids):                              # faces whose pairs fit one chunk
        e = max(s + 1, int(np.searchsorted(ends, (ends[s - 1] if s else 0) + _CHUNK, "right")))
        t, n = ids[s:e], npx[s:e]
        rep = np.repeat(np.arange(len(t)), n)
        k = np.arange(len(rep)) - np.repeat(np.cumsum(n) - n, n)
        dy, dx = k // bw[s:e][rep], k % bw[s:e][rep]
        ti = t[rep]
        px, py = x0[ti] + dx, y0[ti] + dy
        cov, _, _, w = tri_depth(U[ti], V[ti], Wd[ti], px.astype(np.float32), py.astype(np.float32))
        np.minimum.at(zbuf, (py * W + px)[cov], keys(w[cov], ti[cov]))
        s = e
    image = np.broadcast_to(BACKGROUND, (W * H, 3)).copy()
    depth = np.zeros(W * H, np.float32)
    pix = np.nonzero(zbuf != EMPTY)[0]
    t = (zbuf[pix] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    depth[pix] = (zbuf[pix] >> np.uint64(32)).astype(np.uint32).view(np.float32)
    _, q, den, _ = tri_depth(U[t], V[t], Wd[t], (pix % W).astype(np.float32),
                             (pix // W).astype(np.float32))
    f = faces[t]
    shade = face_shade(verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]], eye)
    col = np.asarray(colours, np.uint8).reshape(-1, 3)
    for ch in range(3):
        c = [col[f[:, j], ch].astype(np.float32) for j in range(3)]
        with np.errstate(all="ignore"):
            num = (q[:, 0] * c[0] + q[:, 1] * c[1]) + q[:, 2] * c[2]
            val = np.floor((num / den) * shade + f32(0.5))
        image[pix, ch] = np.fmin(f32(255), np.fmax(f32(0), val)).astype(np.uint8)
    return image.reshape(H, W, 3), depth.reshape(H, W), zbuf


def projected_boxes(verts, faces, P, wh):
    """(drawn mask, box widths, box heights) per face: the kernels rasterise a drawn face in its
    own thread when both are <= SMALL_BOX, else in a CTA."""
    _, _, _, drawn, (x0, x1, y0, y1) = _setup(verts, faces, P, wh)
    return drawn, x1 - x0 + 1, y1 - y0 + 1
