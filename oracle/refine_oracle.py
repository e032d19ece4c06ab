"""Float64 numpy restatement of csrc/refine.cu (casmvsnet_pl_b200/refine.py), with per-element
bounds.  Test infrastructure only.

Steps 1-3 (normals, visibility, selection) and the grey images round every operation as the
kernels do, so they agree bit for bit.  Step 4 projects each patch point X itself, where the kernel
projects by linearity; the two differ only by rounding, and score_bound gives the per-element
bound on S_k that covers it.  Steps 5-6 follow from those.

    out = refine_mesh(verts, faces, images, Ps, sources, iterations)   # dict of every iteration
"""
import numpy as np

from oracle import render_oracle as RO
from oracle import texture_oracle as TO

R, K, STEP, S_MAX, SPACING, MIN_GAIN = 2, 4, 1.0, 4, 4.0, 5e-4
VAR_MIN, MIN_SCORE, LAMBDA, SMOOTH_ROUNDS = 1e-4, 0.3, 1.0, 4
PAD, MIN_COS, DEPTH_SCALE = 2, 0.1, np.float32(1.01)
NO_K = -1000
N = (2 * R + 1) ** 2
EPS = np.finfo(np.float64).eps
# A patch sample's error: the pixel position of a linearised double projection is within about
# 2^-40 px of the direct one at image sides <= 16384 (|q| / w < 2^14, a few roundings of 2^-53
# each, amplified by the coordinates' cancellation), and bilinear grey values in [0, 1] change by
# at most 1 per pixel.
SAMPLE_ERR = 2.0 ** -40


def grey(img):
    c = np.asarray(img, np.uint8).astype(np.float64)
    return ((0.299 * c[..., 0] + 0.587 * c[..., 1]) + 0.114 * c[..., 2]) / 255.0


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def normals(verts, faces):
    """Step 1 -> (V,3) float64."""
    x = np.asarray(verts, np.float32).reshape(-1, 3).astype(np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    e1, e2 = x[f[:, 1]] - x[f[:, 0]], x[f[:, 2]] - x[f[:, 0]]
    fn = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1],
                   e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                   e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    s = np.zeros_like(x)
    np.add.at(s, f.reshape(-1), np.repeat(fn, 3, 0))         # corners in face order
    nn = np.sqrt(_dot(s, s))
    with np.errstate(all="ignore"):
        return np.where(nn[:, None] > 0, s / nn[:, None], 0.0)


def visibility(verts, normal, Ps, whs, zbufs, eyes):
    """Step 2 -> vis (V, n_views) bool."""
    x = np.asarray(verts, np.float32).reshape(-1, 3)
    out = np.zeros((len(x), len(Ps)), bool)
    for j, (P, (W, H), zb, eye) in enumerate(zip(Ps, whs, zbufs, eyes)):
        u, v, w, ok = RO.project(P, x)
        with np.errstate(all="ignore"):
            ok &= (u >= PAD) & (u <= W - 1 - PAD) & (v >= PAD) & (v <= H - 1 - PAD)
        idx = np.nonzero(ok)[0]
        k = zb[np.rint(v[idx]).astype(np.int64) * W + np.rint(u[idx]).astype(np.int64)]
        depth = (k >> np.uint64(32)).astype(np.uint32).view(np.float32)
        ok2 = (k != RO.EMPTY) & (w[idx] <= depth * DEPTH_SCALE)
        d = np.asarray(eye, np.float64)[None] - x[idx].astype(np.float64)
        ok2 &= np.abs(_dot(normal[idx], d)) >= MIN_COS * np.sqrt(_dot(d, d))
        out[idx[ok2], j] = True
    return out


def select(verts, normal, vis, eyes, sources):
    """Step 3 -> (ref (V,) int, src (V, S_MAX) int)."""
    x = np.asarray(verts, np.float32).reshape(-1, 3).astype(np.float64)
    V = len(x)
    cos = np.full((V, len(eyes)), -1.0)
    for j, eye in enumerate(eyes):
        d = np.asarray(eye, np.float64)[None] - x
        cos[:, j] = np.where(vis[:, j], np.abs(_dot(normal, d)) / np.sqrt(_dot(d, d)), -1.0)
    ref = np.full(V, -1, np.int64)
    src = np.full((V, S_MAX), -1, np.int64)
    for v in range(V):
        if not vis[v].any():
            continue
        best = int(np.argmax(cos[v]))                         # first of the largest
        s = [j for j in sources[best] if vis[v, j]][:S_MAX]
        if s:
            ref[v] = best
            src[v, :len(s)] = s
    return ref, src


def frame(n):
    """Tangent frame (t1, t2) (V,3) of unit normals n."""
    ax = np.argmin(np.abs(n), 1)                              # first of the smallest
    a = np.eye(3)[ax]
    c = np.cross(a, n)
    t1 = c / np.sqrt(_dot(c, c))[:, None]
    return t1, np.cross(n, t1)


def _sample(g, P, X):
    """Bilinear samples of g at world points X (..., 3) through P -> (values, valid)."""
    H, W = g.shape
    P = np.asarray(P, np.float32).astype(np.float64)
    q = X @ P[:3, :3].T + P[:3, 3]
    with np.errstate(all="ignore"):
        u, v = q[..., 0] / q[..., 2], q[..., 1] / q[..., 2]
        ok = (q[..., 2] > 0) & (u >= 0) & (u < W - 1) & (v >= 0) & (v < H - 1)
    u, v = np.where(ok, u, 0.0), np.where(ok, v, 0.0)
    fx, fy = np.floor(u), np.floor(v)
    ax, ay = u - fx, v - fy
    x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    c0 = (1 - ax) * g[y0, x0] + ax * g[y0, x1]
    c1 = (1 - ax) * g[y1, x0] + ax * g[y1, x1]
    return (1 - ay) * c0 + ay * c1, ok


def footprint(P, x):
    """rho of points x (V,3) in the view of P (per vertex P (V,4,4) allowed)."""
    P = np.asarray(P, np.float32).astype(np.float64)
    P = np.broadcast_to(P, (len(x), 4, 4))
    q = np.einsum("vij,vj->vi", P[:, :3, :3], x) + P[:, :3, 3]
    z = q[:, 2]
    u, v = q[:, 0] / z, q[:, 1] / z
    Mi = np.linalg.inv(P)
    one = np.ones_like(z)
    a = np.einsum("vij,vj->vi", Mi, np.stack([u * z, v * z, z, one], 1))
    b = np.einsum("vij,vj->vi", Mi, np.stack([(u + 1) * z, v * z, z, one], 1))
    e = a[:, :3] / a[:, 3:] - b[:, :3] / b[:, 3:]
    return np.sqrt(_dot(e, e)), z


def sweep(verts, normal, ref, src, Ps, greys, iteration):
    """Steps 4-5 -> dict: rho, best, kstar, d0, conf (V,), sk (V, 2K+1) NaN where invalid, and
    bound (V, 2K+1), score_bound's per-element bound on sk."""
    x = np.asarray(verts, np.float32).reshape(-1, 3).astype(np.float64)
    V = len(x)
    rho, best = np.zeros(V), np.full(V, np.nan)
    kstar, d0, conf = np.full(V, NO_K, np.int64), np.zeros(V), np.zeros(V)
    sk, bound = np.full((V, 2 * K + 1), np.nan), np.zeros((V, 2 * K + 1))
    Pa = np.stack([np.asarray(P, np.float32) for P in Ps])
    for v in np.nonzero(ref >= 0)[0]:
        r = ref[v]
        rr, z = footprint(Pa[r], x[v:v + 1])
        rho[v] = rr[0]
        if not (z[0] > 0 and rr[0] > 0 and np.isfinite(rr[0])):
            continue
        n = normal[v:v + 1]
        t1, t2 = frame(n)
        step = rho[v] * STEP * 2.0 ** -iteration
        ab = np.arange(-R, R + 1, dtype=np.float64)
        bb, aa = np.meshgrid(ab, ab, indexing="ij")             # row b, column a
        off = SPACING * rho[v] * (aa.reshape(-1, 1) * t1 + bb.reshape(-1, 1) * t2)
        for k in range(-K, K + 1):
            X = x[v] + k * step * n + off                         # (N,3)
            gx, ok = _sample(greys[r], Pa[r], X)
            if not ok.all():
                continue
            mx = gx.sum() / N
            xc = gx - mx
            vx = (xc * xc).sum() / N
            if not vx >= VAR_MIN:
                continue
            zs, cnt, vmin = 0.0, 0, vx
            for j in src[v]:
                if j < 0:
                    continue
                gy, oks = _sample(greys[j], Pa[j], X)
                if not oks.all():
                    continue
                y = gy - mx
                my = y.sum() / N
                vy = (y * y).sum() / N - my * my
                if not vy >= VAR_MIN:
                    continue
                zs += ((xc * y).sum() / N) / np.sqrt(vx * vy)
                cnt += 1
                vmin = min(vmin, vy)
            if cnt:
                sk[v, k + K] = zs / cnt
                bound[v, k + K] = score_bound(vmin)
        kstar[v], best[v], t = choose(sk[v])
        if kstar[v] == NO_K:
            continue
        if sk[v, K] == sk[v, K] and best[v] >= MIN_SCORE:
            conf[v], d0[v] = best[v], (kstar[v] + t) * step
    return dict(rho=rho, best=best, kstar=kstar, d0=d0, conf=conf, sk=sk, bound=bound)


def choose(sk):
    """Step 5's choice over one vertex's scores sk (2K+1,), NaN where k is invalid ->
    (k*, S_k*, t), (NO_K, NaN, 0) without a valid k.  A valid k = 0 stays unless the best k
    beats it by MIN_GAIN; the parabolic sub-step applies to k* != 0 only."""
    kstar, best = NO_K, np.nan
    for k in [0] + [s * m for m in range(1, K + 1) for s in (-1, 1)]:
        s = sk[k + K]
        if s == s and (kstar == NO_K or s > best):
            best, kstar = s, k
    if kstar != NO_K and sk[K] == sk[K] and best - sk[K] < MIN_GAIN:
        kstar, best = 0, sk[K]
    t = 0.0
    if kstar != NO_K and kstar != 0 and -K < kstar < K:
        sm, sp = sk[kstar + K - 1], sk[kstar + K + 1]
        curv = sm - 2 * best + sp
        if sm == sm and sp == sp and curv < 0:
            t = min(max((sm - sp) / (2 * curv), -0.5), 0.5)
    return kstar, best, t


def score_bound(var_min):
    """Bound on |S_k(kernel) - S_k(float64 direct)| when the least population variance among the
    reference and the counting sources is var_min: each sample within SAMPLE_ERR moves a ZNCC by
    at most 2 SAMPLE_ERR / sigma per image (sigma = sqrt(var_min)), and the one-pass variance of
    25 values in [0, 1] adds at most 64 eps / var_min."""
    return 4.0 * SAMPLE_ERR / np.sqrt(var_min) + 64.0 * EPS / var_min


def one_ring(faces, V):
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    a, b = f.reshape(-1), np.roll(f, -1, 1).reshape(-1)
    keep = a != b
    e = np.unique(np.concatenate([(a[keep] << 32) | b[keep], (b[keep] << 32) | a[keep]]))
    lo = e >> 32
    ptr = np.zeros(V + 1, np.int64)
    np.cumsum(np.bincount(lo, minlength=V), out=ptr[1:])
    return ptr, e & 0xFFFFFFFF


def smooth(faces, d0, conf, rounds=SMOOTH_ROUNDS):
    """Step 6's Jacobi rounds -> d (V,)."""
    V = len(d0)
    ptr, ids = one_ring(faces, V)
    cnt = np.diff(ptr).astype(np.float64)
    d = d0.copy()
    for _ in range(rounds):
        s = np.add.reduceat(np.concatenate([d[ids], [0.0]]), np.minimum(ptr[:-1], len(ids)))
        s = np.where(cnt > 0, s, 0.0)
        den = conf + LAMBDA * cnt
        with np.errstate(all="ignore"):
            d = np.where(den > 0, (conf * d0 + LAMBDA * s) / den, 0.0)
    return d


def apply(verts, normal, d):
    x = np.asarray(verts, np.float32).reshape(-1, 3).astype(np.float64)
    return (x + d[:, None] * normal).astype(np.float32)


def refine_mesh(verts, faces, images, Ps, sources, iterations=3):
    """-> dict: verts (final, float32) and per-iteration lists of every step's outputs."""
    Ps = [np.asarray(P, np.float32) for P in Ps]
    greys = [grey(im) for im in images]
    whs = [(g.shape[1], g.shape[0]) for g in greys]
    eyes = [TO.eye_of(P) for P in Ps]
    cur = np.asarray(verts, np.float32).reshape(-1, 3).copy()
    out = dict(iterations=[])
    for it in range(iterations):
        n = normals(cur, faces)
        zbufs = [TO.key_buffer(cur, faces, P, wh) for P, wh in zip(Ps, whs)]
        vis = visibility(cur, n, Ps, whs, zbufs, eyes)
        ref, src = select(cur, n, vis, eyes, sources)
        sw = sweep(cur, n, ref, src, Ps, greys, it)
        d = smooth(faces, sw["d0"], sw["conf"])
        out["iterations"].append(dict(verts=cur, normal=n, vis=vis, ref=ref, src=src, d=d, **sw))
        cur = apply(cur, n, d)
    out["verts"] = cur
    return out


# ---------------------------------------------------------------------------- test scenes
def plane_texture(x, y):
    """A band-limited RGB texture (uint8) of the plane z = 0 at world (x, y): two plane waves per
    channel of periods 0.25 and 0.17."""
    c = []
    for a, b, p in ((1.0, 0.3, 0.0), (0.4, 1.0, 1.0), (0.7, -0.6, 2.0)):
        c.append(0.5 + 0.2 * np.sin(2 * np.pi * (a * x + b * y) / 0.25 + p)
                 + 0.15 * np.sin(2 * np.pi * (b * x - a * y) / 0.17 + 2 * p))
    return np.clip(np.rint(np.stack(c, -1) * 255), 0, 255).astype(np.uint8)


def plane_scene(wh=(160, 120), f=150.0, height=3.0, spread=0.8, constant=None):
    """Five pinhole views of the textured plane z = 0 (plane_texture, or one `constant` RGB
    colour) from (0, 0), (+-spread, 0) and (0, +-spread) at `height`, each aimed at the origin,
    rendered analytically at pixel centres -> (images (H,W,3) uint8, Ps (4,4) float32, sources:
    every other view, in index order)."""
    W, H = wh
    Kc = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1.0]])
    ims, Ps = [], []
    for ox, oy in ((0, 0), (spread, 0), (-spread, 0), (0, spread), (0, -spread)):
        C = np.array([ox, oy, height], np.float64)
        z = -C / np.linalg.norm(C)
        x = np.cross([0.0, 1.0, 0.0], z)
        x /= np.linalg.norm(x)
        Rm = np.stack([x, np.cross(z, x), z])
        P = np.eye(4)
        P[:3, :3], P[:3, 3] = Kc @ Rm, Kc @ (-Rm @ C)
        ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
        r = np.stack([xs, ys, np.ones_like(xs)], -1) @ np.linalg.inv(Kc).T @ Rm
        X = C + (-C[2] / r[..., 2])[..., None] * r
        ims.append(plane_texture(X[..., 0], X[..., 1]) if constant is None else
                   np.broadcast_to(np.asarray(constant, np.uint8), (H, W, 3)).copy())
        Ps.append(P.astype(np.float32))
    return ims, Ps, [[j for j in range(5) if j != i] for i in range(5)]


def grid_mesh(n=16, half=0.35, z=0.0):
    """An n x n vertex grid over [-half, half]^2 at height z -> (verts (n^2,3) float32, faces
    int32)."""
    a = np.linspace(-half, half, n)
    X, Y = np.meshgrid(a, a)
    v = np.stack([X.ravel(), Y.ravel(), np.full(n * n, z)], 1).astype(np.float32)
    q = (np.arange(n - 1)[:, None] * n + np.arange(n - 1)[None]).ravel()
    f = np.concatenate([np.stack([q, q + 1, q + n + 1], 1), np.stack([q, q + n + 1, q + n], 1)])
    return v, f.astype(np.int32)
