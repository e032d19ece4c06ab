"""numpy float64 restatement of csrc/poisson.cu (Poisson surface reconstruction on a dense node
grid), stage by stage: grid, cell moments and normals, orientation, splat, divergence, multigrid,
iso level, trim and colour, then marching cubes through oracle/mesh_oracle.py.  Plus a direct
sparse solve of the same system for small grids.  Dense arrays are (N,N,N) indexed [x, y, z],
which is the kernel's flat layout ((x N + y) N + z) reshaped.  Never imported by the product."""
from __future__ import annotations

import math

import numpy as np
from scipy import ndimage, sparse
from scipy.sparse import linalg as splinalg

from oracle import mesh_oracle

f32 = np.float32
MIN_DEPTH, MAX_DEPTH = 6, 10
RANK_EPS = 1e-10                 # covariance rank < 2 when lambda_mid <= RANK_EPS * lambda_max
COARSEST = 8


def grid(xyz, depth):
    """-> dict(h, N, lo (3,) int64, centre (3,) float64) of the finite points of xyz (n,3)."""
    if not MIN_DEPTH <= depth <= MAX_DEPTH:
        raise ValueError(f"depth must be in {MIN_DEPTH}..{MAX_DEPTH}, got {depth}")
    p = np.asarray(xyz, dtype=f32).reshape(-1, 3)
    p = p[np.isfinite(p).all(1)]
    if not len(p):
        raise ValueError("the cloud has no finite point")
    mn, mx = p.min(0).astype(np.float64), p.max(0).astype(np.float64)
    E = float((mx - mn).max())
    if E == 0:
        raise ValueError("the cloud's bounding box has zero extent")
    N = 1 << depth
    h = float(f32(1.1 * E / N))
    c = (mn + mx) / 2
    lo = np.floor(c / h).astype(np.int64) - N // 2
    return dict(h=h, N=N, lo=lo, centre=c)


def cell_index(p, g):
    """Local node index (n,3) int64 of each point's cell, round(p / h) - lo (float32 division)."""
    q = np.asarray(p, dtype=f32) / f32(g["h"])
    return np.rint(q).astype(np.int64) - g["lo"]


def flat(ijk, N):
    return (ijk[..., 0] * N + ijk[..., 1]) * N + ijk[..., 2]


def estimate_normals(p, g, cams):
    """Unoriented normals of the 3x3x3-cell blocks, oriented toward the nearest camera centre
    (ties to the lower index) -> (normals (n,3) float64, ok (n,) bool)."""
    p = np.asarray(p, dtype=f32)
    N = g["N"]
    key = flat(cell_index(p, g), N)
    cells, inv, cnt = np.unique(key, return_inverse=True, return_counts=True)
    d = p.astype(np.float64) - g["centre"]
    S = np.zeros((len(cells), 3))
    SS = np.zeros((len(cells), 3, 3))
    np.add.at(S, inv, d)
    np.add.at(SS, inv, d[:, :, None] * d[:, None, :])
    cell_of = np.full(N ** 3, -1, np.int64)
    cell_of[cells] = np.arange(len(cells))
    cijk = np.stack([cells // (N * N), (cells // N) % N, cells % N], 1)
    n_t, S_t, SS_t = np.zeros(len(cells)), np.zeros((len(cells), 3)), np.zeros((len(cells), 3, 3))
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dz in (-1, 0, 1):
                q = cijk + np.array([dx, dy, dz])
                inside = ((q >= 0) & (q < N)).all(1)
                nb = np.full(len(cells), -1)
                nb[inside] = cell_of[flat(q[inside], N)]
                m = nb >= 0
                n_t[m] += cnt[nb[m]]
                S_t[m] += S[nb[m]]
                SS_t[m] += SS[nb[m]]
    with np.errstate(all="ignore"):
        mu = S_t / n_t[:, None]
        cov = SS_t / n_t[:, None, None] - mu[:, :, None] * mu[:, None, :]
    cov = np.where(n_t[:, None, None] >= 3, cov, np.eye(3))
    lam, vec = np.linalg.eigh(cov)
    ok_c = (n_t >= 3) & (lam[:, 2] > 0) & (lam[:, 1] > RANK_EPS * lam[:, 2])
    nc = vec[:, :, 0]
    nc = nc / np.linalg.norm(nc, axis=1, keepdims=True)
    n = nc[inv]
    cams = np.asarray(cams, dtype=np.float64).reshape(-1, 3)
    pd = p.astype(np.float64)
    d2 = ((pd[:, None, :] - cams[None]) ** 2).sum(-1)
    C = cams[np.argmin(d2, axis=1)]
    flip = (n * (C - pd)).sum(1) < 0
    n[flip] = -n[flip]
    return n, ok_c[inv]


def normalise(normals):
    """PLY normals -> (unit normals float64, ok) ; zero-length or non-finite ones are not ok."""
    n = np.asarray(normals, dtype=f32).astype(np.float64)
    L = np.sqrt((n * n).sum(1))
    ok = np.isfinite(L) & (L > 0)
    with np.errstate(all="ignore"):
        return np.where(ok[:, None], n / L[:, None], 0.0), ok


def _corners(p, g):
    """-> (base (n,3) local node of floor(p/h), frac (n,3) float32)."""
    q = np.asarray(p, dtype=f32) / f32(g["h"])
    fl = np.floor(q)
    return fl.astype(np.int64) - g["lo"], (q - fl).astype(f32)


def trilinear(frac, d):
    """float32 weight of corner d = (dx, dy, dz) in {0,1}^3: (wx wy) wz."""
    w = [frac[:, a] if d[a] else f32(1) - frac[:, a] for a in range(3)]
    return (w[0] * w[1]) * w[2]


CORNERS = [(dx, dy, dz) for dx in (0, 1) for dy in (0, 1) for dz in (0, 1)]


def splat(p, n, rgb, g):
    """-> V (N,N,N,3), W (N,N,N), C (N,N,N,3), float64 sums of the float32 trilinear weights."""
    N = g["N"]
    base, frac = _corners(p, g)
    n = np.asarray(n, dtype=f32).astype(np.float64)
    rgb = np.asarray(rgb, dtype=np.float64)
    V, W, C = np.zeros((N ** 3, 3)), np.zeros(N ** 3), np.zeros((N ** 3, 3))
    for d in CORNERS:
        w = trilinear(frac, d).astype(np.float64)
        idx = flat(base + np.array(d), N)
        np.add.at(W, idx, w)
        np.add.at(V, idx, w[:, None] * n)
        np.add.at(C, idx, w[:, None] * rgb)
    return V.reshape(N, N, N, 3), W.reshape(N, N, N), C.reshape(N, N, N, 3)


def divergence(V, h):
    """b = div V by central differences at the interior nodes, 0 on the outer layer."""
    b = np.zeros(V.shape[:3])
    i = slice(1, -1)
    b[i, i, i] = (((V[2:, i, i, 0] - V[:-2, i, i, 0]) + (V[i, 2:, i, 1] - V[i, :-2, i, 1]))
                  + (V[i, i, 2:, 2] - V[i, i, :-2, 2])) / (2 * h)
    return b


def _nbsum(e):
    s = np.zeros_like(e)
    i = slice(1, -1)
    s[i, i, i] = ((((e[:-2, i, i] + e[2:, i, i]) + e[i, :-2, i]) + e[i, 2:, i]) + e[i, i, :-2]) + e[i, i, 2:]
    return s


def _interior(n):
    m = np.zeros((n, n, n), bool)
    m[1:-1, 1:-1, 1:-1] = True
    return m


def apply_laplacian(x, h):
    """(sum of the 6 neighbours - 6 x) / h^2 at interior nodes, 0 on the outer layer."""
    return np.where(_interior(len(x)), (_nbsum(x) - 6 * x) / (h * h), 0.0)


def _smooth(e, r, h, sweeps):
    n = len(e)
    ii = np.indices((n, n, n)).sum(0)
    inner = _interior(n)
    for _ in range(sweeps):
        for parity in (0, 1):
            m = inner & (ii % 2 == parity)
            e[m] = ((_nbsum(e) - h * h * r) / 6)[m]
    return e


def _restrict_1d(a, axis):
    a = np.moveaxis(a, axis, 0)
    nc = len(a) // 2
    out = np.zeros((nc + 1,) + a.shape[1:])
    I = np.arange(1, nc)
    out[I] = 0.25 * a[2 * I - 1] + 0.5 * a[2 * I] + 0.25 * a[2 * I + 1]
    return np.moveaxis(out, 0, axis)


def restrict(r):
    """Full weighting of a level's residual onto the next coarser level.  A level of n nodes per
    axis (n = N >> l) is stored with n + 1 array entries when it is coarse: entry n is the zero
    Dirichlet node at fine index N, the same place on every coarse level, so the coarse interior
    is 1..n-1.  Coarse interior node I takes fine 2I + {-1,0,1}, weights (1/4, 1/2, 1/4)."""
    for a in range(3):
        r = _restrict_1d(r, a)
    return r


def _prolong_1d(a, axis, m):
    a = np.moveaxis(a, axis, 0)
    out = np.empty((m,) + a.shape[1:])
    out[0::2] = a[:(m + 1) // 2]
    k = np.arange(m // 2)
    out[1::2] = 0.5 * (a[k] + a[k + 1])
    return np.moveaxis(out, 0, axis)


def prolong(e, m):
    """Trilinear interpolation of coarse node I (at fine 2I) onto the m^3 fine array entries."""
    for a in range(3):
        e = _prolong_1d(e, a, m)
    return e


def vcycle(r, h, pre=2, post=2, coarse_sweeps=50):
    """One V(pre, post) cycle for L e = r from e = 0, red-black Gauss-Seidel, coarsening to
    COARSEST^3 nodes, where coarse_sweeps sweeps are run.  r is the finest level (N^3, outer layer
    Dirichlet) or a coarse level ((n + 1)^3, see restrict)."""
    m = len(r)
    e = np.zeros_like(r)
    if m - m % 2 <= COARSEST:
        return _smooth(e, r, h, coarse_sweeps)
    _smooth(e, r, h, pre)
    res = np.where(_interior(m), r - apply_laplacian(e, h), 0.0)
    ec = vcycle(restrict(res), 2 * h, pre, post, coarse_sweeps)
    e += np.where(_interior(m), prolong(ec, m), 0.0)
    return _smooth(e, r, h, post)


def norm2(x):
    return math.sqrt(float((np.asarray(x, np.float64) ** 2).sum()))


def multigrid(b, h, tol=1e-5, max_cycles=40):
    """Solve L chi = b, chi = 0 on the outer layer: V(2,2) cycles until ||r|| / ||b|| <= tol or
    max_cycles cycles -> (chi, cycles, ratio)."""
    chi = np.zeros_like(b)
    bn = norm2(b)
    if bn == 0:
        return chi, 0, 0.0
    cycles = 0
    while True:
        r = np.where(_interior(len(b)), b - apply_laplacian(chi, h), 0.0)
        ratio = norm2(r) / bn
        if ratio <= tol or cycles == max_cycles:
            return chi, cycles, ratio
        chi += vcycle(r, h)
        cycles += 1


def direct_solve(b, h):
    """The same Dirichlet system solved with scipy.sparse.linalg.spsolve (small grids only)."""
    n = len(b)
    m = n - 2
    one = sparse.identity(m, format="csr")
    t = sparse.diags([np.ones(m - 1), -2 * np.ones(m), np.ones(m - 1)], [-1, 0, 1], format="csr")
    A = (sparse.kron(sparse.kron(t, one), one) + sparse.kron(sparse.kron(one, t), one)
         + sparse.kron(sparse.kron(one, one), t)) / (h * h)
    x = splinalg.spsolve(A.tocsc(), b[1:-1, 1:-1, 1:-1].reshape(-1))
    chi = np.zeros_like(b)
    chi[1:-1, 1:-1, 1:-1] = x.reshape(m, m, m)
    return chi


def iso_level(chi, p, g):
    """Mean over the points of chi trilinearly interpolated (float32 weights, float64 sums)."""
    base, frac = _corners(p, g)
    N = g["N"]
    v = np.zeros(len(base))
    c = chi.reshape(-1)
    for d in CORNERS:
        v += trilinear(frac, d).astype(np.float64) * c[flat(base + np.array(d), N)]
    return float(v.sum() / len(v))


def trim(W):
    """Kept nodes: the 5x5x5 box sum of W around the node is positive."""
    return ndimage.maximum_filter((W > 0).astype(np.uint8), size=5, mode="constant") > 0


def box5(a):
    k = np.ones((5, 5, 5))
    if a.ndim == 4:
        return np.stack([ndimage.convolve(a[..., c], k, mode="constant") for c in range(3)], -1)
    return ndimage.convolve(a, k, mode="constant")


def colour(C, W, keep):
    Wb, Cb = box5(W), box5(C)
    with np.errstate(all="ignore"):
        return np.where(keep[..., None], Cb / Wb[..., None], 0.0)


def bricks(f, keep, col, g):
    """The kept nodes in mesh.cu's brick layout -> (keys, tsdf, weight, color) float32."""
    N, lo = g["N"], g["lo"]
    ijk = np.argwhere(keep) + lo
    keys = np.unique(mesh_oracle.pack_keys(ijk // 8))
    gi = mesh_oracle.voxel_indices(keys) - lo
    inside = ((gi >= 0) & (gi < N)).all(1)
    sel = np.zeros(len(gi), bool)
    sel[inside] = keep[tuple(gi[inside].T)]
    tsdf = np.zeros(len(gi), f32)
    weight = np.zeros(len(gi), f32)
    color = np.zeros((len(gi), 3), f32)
    t = tuple(gi[sel].T)
    tsdf[sel], weight[sel], color[sel] = f[t], 1, col[t]
    return keys, tsdf, weight, color


def poisson(xyz, rgb=None, normals=None, cams=None, depth=9, tol=1e-5, max_cycles=40):
    """Every stage -> dict (grid, kept points, their normals, V, W, C, b, chi, cycles, ratio, iso,
    keep, colour, keys, tsdf, weight, color, verts, colours, faces, dropped, kept (input mask))."""
    p = np.asarray(xyz, dtype=f32).reshape(-1, 3)
    g = grid(p, depth)
    ok = np.isfinite(p).all(1)
    if normals is not None:
        n, okn = normalise(normals)
        ok &= okn
    else:
        if cams is None:
            raise ValueError("a cloud without normals needs camera centres")
        n = np.zeros((len(p), 3))
        n[ok], okn = estimate_normals(p[ok], g, cams)
        ok[np.nonzero(ok)[0][~okn]] = False
    rgb = np.full((len(p), 3), 255.0) if rgb is None else np.asarray(rgb, np.float64)
    pk, nk, ck = p[ok], n[ok].astype(f32), rgb[ok]
    V, W, C = splat(pk, nk, ck, g)
    b = divergence(V.astype(f32).astype(np.float64), g["h"])
    chi, cycles, ratio = multigrid(b, g["h"], tol, max_cycles)
    iso = iso_level(chi, pk, g)
    keep = trim(W)
    col = colour(C.astype(f32).astype(np.float64), W.astype(f32).astype(np.float64), keep)
    f = chi - iso
    keys, tsdf, weight, color = bricks(f, keep, col, g)
    verts, colours, faces = mesh_oracle.extract(keys, tsdf, weight, color, g["h"])
    return dict(grid=g, points=pk, normals=nk, V=V, W=W, C=C, b=b, chi=chi, cycles=cycles,
                ratio=ratio, iso=iso, keep=keep, colour=col, keys=keys, tsdf=tsdf, weight=weight,
                color=color, verts=verts, colours=colours, faces=faces, dropped=int((~ok).sum()),
                kept=ok)


# ------------------------------------------------------------------------------ test clouds
def sphere(n, radius=1.0, seed=0, noise=0.0):
    """n points on a sphere (Fibonacci lattice, seeded rotation), exact outward normals, radial
    noise of standard deviation `noise` -> (xyz float32, normals float32)."""
    rng = np.random.default_rng(seed)
    i = np.arange(n) + 0.5
    z = 1 - 2 * i / n
    az = i * np.pi * (3 - np.sqrt(5))
    u = np.stack([np.sqrt(1 - z * z) * np.cos(az), np.sqrt(1 - z * z) * np.sin(az), z], 1)
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    u = u @ q
    r = radius + noise * rng.normal(size=(n, 1))
    return (u * r).astype(f32), u.astype(f32)


def plane(n, size=1.0, seed=0, noise=0.0):
    """n points on the square |x|, |y| <= size / 2 of z = 0 with z noise, normals +z."""
    rng = np.random.default_rng(seed)
    p = np.concatenate([rng.uniform(-size / 2, size / 2, (n, 2)), noise * rng.normal(size=(n, 1))], 1)
    nrm = np.tile([0.0, 0.0, 1.0], (n, 1))
    return p.astype(f32), nrm.astype(f32)
