"""The Poisson float64 reference (oracle/poisson_fp64.py) without a GPU: it agrees with scipy and
numpy float64, a float32 restatement of every kernel passes every bound at every element at
depths 6-8 and at |p/h| up to the grid's 2^23 guard, and each defect injected into that
restatement fails with the report pointing at the defect."""
import numpy as np
import pytest
import torch
from scipy import ndimage

from oracle import poisson_fp64 as F
from oracle import poisson_oracle as O

f32 = torch.float32


# ------------------------------------------------------------------------------- float32 restatement
# Each function mirrors one kernel of csrc/poisson.cu operation for operation (float32 where the
# kernel is float32, double where it is double); `defect` switches in one subtle error.
def _pad0(e):
    n = e.shape[0]
    P = torch.zeros(n + 2, n + 2, n + 2, dtype=e.dtype)
    P[1:-1, 1:-1, 1:-1] = e
    return P


def _nbsum(P):
    i = slice(1, -1)
    return (((((P[:-2, i, i] + P[2:, i, i]) + P[i, :-2, i]) + P[i, 2:, i]) + P[i, i, :-2])
            + P[i, i, 2:])


def _inner(n, level):
    return F.interior(F.full(n), n, level, "cpu")


def smooth32(e, r, level, h, sweeps=1, zero_first=False, defect=None):
    n = e.shape[0]
    e = torch.zeros_like(e) if zero_first else e.clone()
    h2 = torch.tensor(h, dtype=f32) * torch.tensor(h, dtype=f32)
    x, y, z = F._grid_xyz(F.full(n), "cpu")
    par = (x + y + z) % 2
    order = (1, 0) if defect == "black_first" else (0, 1)
    for _ in range(sweeps):
        for parity in order:
            m = _inner(n, level) & (par == parity)
            e = torch.where(m, (_nbsum(_pad0(e)) - h2 * r) / 6, e)
    return e


def mg_residual32(e, r, level, h):
    n = e.shape[0]
    h2 = torch.tensor(h, dtype=f32) * torch.tensor(h, dtype=f32)
    out = r - (_nbsum(_pad0(e)) - 6 * e) / h2
    return torch.where(_inner(n, level), out, torch.zeros_like(out))


def restrict32(f, defect=None):
    nf = f.shape[0]
    nc = nf // 2
    P = torch.zeros(nf + 1, nf + 1, nf + 1, dtype=f32)
    P[1:, 1:, 1:] = f                                          # fine index -1 -> entry 0
    wx = {"restrict_third": (1 / 3, 1 / 3, 1 / 3),
          "restrict_half": (0.125, 0.25, 0.125)}.get(defect, (0.25, 0.5, 0.25))
    s = torch.zeros(nc, nc, nc, dtype=f32)
    I = torch.arange(nc)
    for a, dx in enumerate((-1, 0, 1)):
        for b, dy in enumerate((-1, 0, 1)):
            for c, dz in enumerate((-1, 0, 1)):
                w = torch.tensor(wx[a] * (0.25, 0.5, 0.25)[b] * (0.25, 0.5, 0.25)[c], dtype=f32)
                X, Y, Z = ((2 * I + d + 1).clamp(0, nf) for d in (dx, dy, dz))
                s = s + w * P[X][:, Y][:, :, Z]
    return torch.where(_inner(nc, 1), s, torch.zeros_like(s))


def prolong_add32(c, f, fine_level, defect=None):
    nc = c.shape[0]
    nf = 2 * nc
    C = torch.zeros(nc + 1, nc + 1, nc + 1, dtype=f32)
    C[:nc, :nc, :nc] = c
    if defect == "prolong_stored_n":                           # index nc reads the stored nc - 1
        C[nc, :, :] = C[nc - 1, :, :]
        C[:, nc, :] = C[:, nc - 1, :]
        C[:, :, nc] = C[:, :, nc - 1]
    p = torch.arange(nf)
    i0, i1 = p >> 1, (p + 1) >> 1
    w1 = torch.where(p % 2 == 1, 0.5, 0.0).to(f32)
    s = torch.zeros(nf, nf, nf, dtype=f32)
    for d in range(8):
        dx, dy, dz = d >> 2, (d >> 1) & 1, d & 1
        wa = [w1 if dd else 1 - w1 for dd in (dx, dy, dz)]
        w = (wa[0][:, None, None] * wa[1][None, :, None]) * wa[2][None, None, :]
        X, Y, Z = (i1 if dx else i0), (i1 if dy else i0), (i1 if dz else i0)
        s = s + w * C[X][:, Y][:, :, Z]
    return torch.where(_inner(nf, fine_level), f + s, f)


def residual64(chi, b, h):
    n = chi.shape[0]
    hh = float(np.float32(h)) ** 2
    r = b.double() - (_nbsum(_pad0(chi)) - 6.0 * chi) / hh
    r = torch.where(_inner(n, 0), r, torch.zeros_like(r))
    return r.float(), float((r * r).sum())


def rhs32(V, h):
    n = V.shape[0]
    P = torch.zeros(n + 2, n + 2, n + 2, 3, dtype=torch.float64)
    P[1:-1, 1:-1, 1:-1] = V.double()
    i = slice(1, -1)
    d = ((P[2:, i, i, 0] - P[:-2, i, i, 0]) + (P[i, 2:, i, 1] - P[i, :-2, i, 1])) + \
        (P[i, i, 2:, 2] - P[i, i, :-2, 2])
    b = torch.where(_inner(n, 0), (d / (2.0 * float(np.float32(h)))), torch.zeros_like(d)).float()
    return b, float((b.double() ** 2).sum())


def cell_keys32(p, h, lo, N, defect=None):
    q = torch.from_numpy(p) / torch.tensor(np.float32(h))
    c = torch.floor(q + 0.5) if defect == "floor_half" else torch.round(q)
    ok = torch.isfinite(c).all(1) & (c.abs() < 1e9).all(1)
    c = torch.where(torch.isfinite(c), c, torch.zeros_like(c)).long() - torch.tensor(lo)
    ok &= ((c >= 0) & (c < N)).all(1)
    return torch.where(ok, (c[:, 0] * N + c[:, 1]) * N + c[:, 2], torch.tensor(F.KEY_NONE))


def splat32(p, n, rgb, h, lo, N, defect=None):
    p = torch.from_numpy(p)
    q = p / torch.tensor(np.float32(h))
    fl = torch.floor(q)
    fr = q - fl
    base = fl.long() - torch.tensor(lo)
    cell = torch.round(q).long() - torch.tensor(lo)
    n = torch.from_numpy(n).double()
    col = torch.full_like(n, 255.0) if rgb is None else torch.from_numpy(rgb).double()
    W = torch.zeros(N ** 3, dtype=torch.float64)
    V = torch.zeros(N ** 3, 3, dtype=torch.float64)
    C = torch.zeros(N ** 3, 3, dtype=torch.float64)
    for d in O.CORNERS:
        w = [fr[:, a] if d[a] else 1 - fr[:, a] for a in range(3)]
        wt = ((w[0] * w[1]) * w[2]).double()
        node = base + torch.tensor(d)
        ok = ((node >= 0) & (node < N)).all(1)
        if defect == "skip_27th":                             # the cell at node + (1, 1, 1)
            ok &= ~(cell - node == 1).all(1)
        idx = ((node[:, 0] * N + node[:, 1]) * N + node[:, 2])[ok]
        W.index_add_(0, idx, wt[ok])
        V.index_add_(0, idx, wt[ok, None] * n[ok])
        C.index_add_(0, idx, wt[ok, None] * col[ok])
    return (V.float().reshape(N, N, N, 3), W.float().reshape(N, N, N), C.float().reshape(N, N, N, 3))


def iso32(chi, p, h, lo, N, defect=None):
    terms = F.iso_terms(chi, p, h, lo, N)
    if defect == "iso_float":
        s = torch.zeros((), dtype=f32)
        for v in terms.sum(1).float():
            s = s + v
        return float(s)
    return float(terms.sum())


def trim32(W, radius=2):
    m = (W > 0).numpy().astype(np.uint8)
    return torch.from_numpy(ndimage.maximum_filter(m, size=2 * radius + 1, mode="constant"))


def normals32(ckeys, mom, N, defect=None):
    M = F.block_moments(ckeys, mom, N).numpy()
    m0 = M[:, 0]
    with np.errstate(all="ignore"):
        mu = M[:, 1:4] / m0[:, None]
        cov = np.empty((len(M), 3, 3))
        for a, b, j in [(0, 0, 4), (0, 1, 5), (0, 2, 6), (1, 1, 7), (1, 2, 8), (2, 2, 9)]:
            cov[:, a, b] = cov[:, b, a] = M[:, j] / m0 - mu[:, a] * mu[:, b]
    few = m0 < 3
    cov[few] = np.eye(3)
    lam, vec = np.linalg.eigh(cov)
    ok = ~few & (lam[:, 2] > 0) & (lam[:, 1] > F.RANK_EPS * lam[:, 2])
    v = vec[:, :, 2] if defect == "eig_order" else vec[:, :, 0]
    return torch.from_numpy(np.where(ok[:, None], v, 0.0)), torch.from_numpy(ok.astype(np.uint8))


def orient32(p, pcell, cn, cams, defect=None):
    pd = torch.from_numpy(p).double()
    cams = torch.as_tensor(cams, dtype=torch.float64)
    best = torch.full((len(p),), float("inf"), dtype=torch.float64)
    kb = torch.zeros(len(p), dtype=torch.long)
    for k in range(len(cams)):
        d = pd - cams[k]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        take = d2 <= best if defect == "tie_high" else d2 < best
        best = torch.where(take, d2, best)
        kb = torch.where(take, torch.full_like(kb, k), kb)
    n = cn[pcell]
    dot = (n * (cams[kb] - pd)).sum(1)
    return torch.where((dot < 0)[:, None], -n, n).float()


def vcycle32(r, hs, level=0, defect=None):
    n = r.shape[0]
    if n <= F.COARSEST:
        return smooth32(torch.zeros_like(r), r, level, hs[level], 50, True)
    e = smooth32(torch.zeros_like(r), r, level, hs[level], 2, True)
    res = mg_residual32(e, r, level, hs[level])
    ec = vcycle32(restrict32(res, defect), hs, level + 1, defect)
    e = prolong_add32(ec, e, level)
    return smooth32(e, r, level, hs[level], 2)


def multigrid32(b, h, defect=None, tol=1e-5):
    N = b.shape[0]
    hs = F.hs_levels(h, N)
    chi = torch.zeros(N, N, N, dtype=torch.float64)
    bn = float((b.double() ** 2).sum()) ** 0.5
    ratios = []
    while True:
        r, rr = residual64(chi, b, h)
        ratios.append(rr ** 0.5 / bn)
        if ratios[-1] <= tol or len(ratios) > 40:
            return chi, ratios
        chi = chi + vcycle32(r, hs, 0, defect).double()


# ------------------------------------------------------------------------------- inputs
def _grid(depth, offset=0.0, n=4000, seed=0):
    p, nrm = O.sphere(n, seed=seed, noise=0.01)
    p = (p.astype(np.float64) + offset).astype(np.float32)
    return p, nrm, O.grid(p, depth)


def _lo(g):
    return [int(v) for v in g["lo"]]


def _fields(depth, seed=0):
    """A real right-hand side (a sphere splatted at this depth) and seeded random fields."""
    p, nrm, g = _grid(depth, n=3000, seed=seed)
    N, h = g["N"], g["h"]
    V, W, C = splat32(p, nrm, None, h, _lo(g), N)
    b, _ = rhs32(V, h)
    rng = np.random.default_rng(seed)
    rand = lambda n: torch.from_numpy(rng.standard_normal((n, n, n)).astype(np.float32))
    return g, b, rand


def _wins(n, depth):
    return None if depth <= 7 else F.windows(n, 24)


# ------------------------------------------------------------------------------- fp64 vs scipy, numpy
def test_fp64_laplacian_and_multigrid_agree_with_the_direct_solve():
    p, n = O.sphere(3000, seed=1)
    N = 32
    h = float(np.float32(1.1 * 2 / N))
    g = dict(h=h, N=N, lo=np.full(3, -N // 2, np.int64), centre=np.zeros(3))
    V, _, _ = O.splat(p, n, np.full((len(p), 3), 255.0), g)
    b = O.divergence(V, h)
    direct = O.direct_solve(b, h)
    Lx = F.laplacian(torch.from_numpy(direct), h).numpy()
    assert np.abs(Lx - b).max() <= 1e-12 * np.abs(b).max() * N * N
    chi, ratios = F.multigrid64(torch.from_numpy(b), h, tol=1e-13, max_cycles=60)
    assert ratios[-1] <= 1e-13
    assert np.abs(chi.numpy() - direct).max() <= 1e-10 * np.abs(direct).max()
    # the same V cycle as the numpy restatement's float64 path, its (n + 1) coarse layout aside
    r = torch.from_numpy(b)
    e64 = F.vcycle64(r, float(np.float32(h)))
    eo = O.vcycle(b, float(np.float32(h)))
    assert np.abs(e64.numpy() - eo).max() <= 1e-12 * np.abs(eo).max()


def test_fp64_restrict_and_prolong_agree_with_numpy():
    rng = np.random.default_rng(0)
    f = rng.standard_normal((32, 32, 32))
    f[0], f[-1], f[:, 0], f[:, -1], f[:, :, 0], f[:, :, -1] = 0, 0, 0, 0, 0, 0
    want = O.restrict(f)[:16, :16, :16]
    got = F._ref_restrict(torch.from_numpy(f)).numpy()
    assert np.abs(np.where(F.interior(F.full(16), 16, 1, "cpu").numpy(), got, 0) - want).max() <= 1e-12
    c = rng.standard_normal((16, 16, 16))
    co = np.zeros((17, 17, 17))
    co[:16, :16, :16] = c
    assert np.abs(F._ref_prolong(torch.from_numpy(c)).numpy() - O.prolong(co, 32)).max() <= 1e-12


def test_fp64_normals_trim_and_box_agree_with_numpy_and_ndimage():
    p, _ = O.sphere(20_000, seed=2, noise=0.001)
    g = O.grid(p, 6)
    N = g["N"]
    key = O.flat(O.cell_index(p, g), N)
    order = np.argsort(key, kind="stable")
    ps, ks = p[order], key[order]
    cells, start = np.unique(ks, return_index=True)
    start = np.append(start, len(ks)).astype(np.int32)
    d = ps.astype(np.float64) - g["centre"]
    x, y, z = d.T
    t = np.stack([np.ones_like(x), x, y, z, x * x, x * y, x * z, y * y, y * z, z * z], 1)
    mom = np.add.reduceat(t, start[:-1], axis=0)
    cn, cok = normals32(torch.from_numpy(cells), torch.from_numpy(mom), N)
    want, ok = O.estimate_normals(p, g, [[0, 0, 0]])              # np.linalg.eigh, np.add.at
    inv = np.searchsorted(cells, key)
    assert np.array_equal(cok.numpy()[inv].astype(bool), ok)
    dots = np.abs((cn.numpy()[inv] * want).sum(1))
    assert np.abs(dots - 1).max() <= 1e-12
    rep = F.check_normals(cells, mom, N, cn, cok)
    assert rep.ok, rep.describe()
    W = torch.zeros(N, N, N)
    rng = np.random.default_rng(1)
    W.view(-1)[torch.from_numpy(rng.choice(N ** 3, 300, replace=False))] = 1.0
    assert F.check_trim(W, trim32(W), N).ok
    a = rng.random((20, 20, 20))
    P = torch.from_numpy(np.pad(a, 2))
    want = ndimage.convolve(a, np.ones((5, 5, 5)), mode="constant")
    assert np.abs(F.box5(P).numpy() - want).max() <= 1e-12 * np.abs(want).max()


# ------------------------------------------------------------------------------- restatement passes
def _check_levels(depth, defect=None):
    """Every multigrid kernel of the restatement at every level -> dict of reports."""
    g, b, rand = _fields(depth)
    N, h = g["N"], g["h"]
    hs = F.hs_levels(h, N)
    reps = {}
    chi = rand(N).double() * 1e-3
    r, rr = residual64(chi, b, h)
    wins = _wins(N, depth)
    reps["residual"], parts = F.check_residual(chi, b, r, N, h, wins)
    Vr = torch.from_numpy(np.stack([rand(N).numpy() for _ in range(3)], -1))
    bb_b, bb = rhs32(Vr, h)
    reps["rhs"] = F.check_rhs(Vr, bb_b, N, h, wins)
    reps["reduction"] = F.check_reduction(bb, bb_b.double() ** 2)
    e = rand(N)
    acc = chi + e.double()
    reps["accumulate"] = F.check_accumulate(chi, e, acc, N, wins)
    rhs = [r]
    for l, n in enumerate([N >> k for k in range(len(hs))]):
        wins = _wins(n, depth)
        rl = rhs[l] if l < len(rhs) else rand(n)
        e0 = rand(n) * 1e-2
        for zf in (False, True):
            e1 = smooth32(e0, rl, l, hs[l], 1, zf, defect)
            F.check_smooth(e0, e1, rl, n, l, hs[l], wins, reps.setdefault("smooth", F.Report("smooth")),
                           zero_first=zf)
        out = mg_residual32(e0, rl, l, hs[l])
        F.check_mg_residual(e0, rl, out, n, l, hs[l], wins,
                            reps.setdefault("mg_residual", F.Report("mg_residual")))
        if n > F.COARSEST:
            c = restrict32(out, defect)
            F.check_restrict(out, c, n, l + 1, _wins(n // 2, depth),
                             reps.setdefault("restrict", F.Report("restrict")))
            rhs.append(c)
            ec = rand(n // 2)
            f1 = prolong_add32(ec, e0, l, defect)
            F.check_prolong_add(ec, e0, f1, n // 2, l, wins,
                                reps.setdefault("prolong_add", F.Report("prolong_add")))
    return reps


@pytest.mark.parametrize("depth", [6, 7, 8])
def test_restatement_passes_every_multigrid_bound(depth):
    reps = _check_levels(depth)
    for k, rep in reps.items():
        assert rep.ok, rep.describe()
        assert rep.checked > 0


@pytest.mark.parametrize("offset", [0.0, 1e4, 1e5, 1e6, 4e6, 8.3e6])
def test_restatement_passes_the_point_bounds_far_from_the_origin(offset):
    """cell_keys, splat and iso at |p/h| up to 8.3e6 (the guard is 2^23 ~ 8.4e6): the bounds
    scale with ulp(p/h), so the coarse float32 quotient still passes."""
    depth = 6
    p, nrm, g = _grid(depth, n=3000)
    h = g["h"]
    p = (p.astype(np.float64) + offset * h).astype(np.float32)
    g = O.grid(p, depth)
    N, h, lo = g["N"], g["h"], _lo(g)
    keys = cell_keys32(p, h, lo, N)
    rep, _ = F.check_cell_keys(p, nrm, h, lo, N, keys)
    assert rep.ok, rep.describe()
    ok = keys != F.KEY_NONE
    V, W, C = splat32(p[ok.numpy()], nrm[ok.numpy()], None, h, lo, N)
    reps = F.check_splat(p[ok.numpy()], nrm[ok.numpy()], None, h, lo, N, V, W, C)
    for r in reps.values():
        assert r.ok, r.describe()
    rng = np.random.default_rng(0)
    chi = torch.from_numpy(rng.standard_normal(N ** 3))
    s = iso32(chi, p[ok.numpy()], h, lo, N)
    rep, rep_sum = F.check_iso(chi, p[ok.numpy()], h, lo, N, s)
    assert rep.ok and rep_sum.ok, (rep.describe(), rep_sum.describe())


# ------------------------------------------------------------------------------- injected defects
@pytest.mark.parametrize("defect", ["restrict_third", "restrict_half"])
def test_defect_restrict_weights(defect):
    reps = _check_levels(6, defect)
    rep = reps["restrict"]
    assert not rep.ok and rep.where[0] >= 1, rep.describe()
    assert all(r.ok for k, r in reps.items() if k != "restrict")


def test_defect_prolong_reads_coarse_n_as_stored():
    reps = _check_levels(6, "prolong_stored_n")
    rep = reps["prolong_add"]
    assert not rep.ok, rep.describe()
    level, x, y, z = rep.where
    nf = 64 >> level
    assert nf - 1 in (x, y, z) and level >= 1, rep.describe()   # the coarse level's upper face
    assert all(r.ok for k, r in reps.items() if k != "prolong_add")


def test_defect_black_before_red():
    reps = _check_levels(6, "black_first")
    rep = reps["smooth"]
    assert not rep.ok and sum(rep.where[1:]) % 2 == 0, rep.describe()   # red node: stale input
    assert all(r.ok for k, r in reps.items() if k != "smooth")


def test_defect_splat_skips_the_27th_cell():
    p, nrm, g = _grid(6, n=3000)
    N, h, lo = g["N"], g["h"], _lo(g)
    V, W, C = splat32(p, nrm, None, h, lo, N, "skip_27th")
    reps = F.check_splat(p, nrm, None, h, lo, N, V, W, C)
    rep = reps["W"]
    assert not rep.ok, rep.describe()
    _, x, y, z = rep.where
    # a point of cell (x + 1, y + 1, z + 1) whose floor corner is the node was skipped
    cell = O.cell_index(p, g)
    base, _ = O._corners(p, g)
    hit = (cell == [x + 1, y + 1, z + 1]).all(1) & (base == [x, y, z]).all(1)
    assert hit.any(), rep.describe()


def test_defect_trim_radius_one():
    p, nrm, g = _grid(6, n=3000)
    N, h, lo = g["N"], g["h"], _lo(g)
    _, W, _ = splat32(p, nrm, None, h, lo, N)
    rep = F.check_trim(W, trim32(W, 1), N)
    assert not rep.ok, rep.describe()
    _, x, y, z = rep.first_bad
    d = ndimage.distance_transform_cdt((W.numpy() <= 0).astype(np.uint8), metric="chessboard")
    assert d[x, y, z] == 2, rep.describe()                      # 2 nodes from the nearest W > 0


def test_defect_float32_iso_sum():
    p, nrm, g = _grid(6, n=20_000)
    N, h, lo = g["N"], g["h"], _lo(g)
    chi = torch.from_numpy(np.random.default_rng(0).standard_normal(N ** 3) + 3.0)
    rep, rep_sum = F.check_iso(chi, p, h, lo, N, iso32(chi, p, h, lo, N, "iso_float"))
    assert rep.ok and not rep_sum.ok and rep_sum.where[0] == "sum", rep_sum.describe()
    _, ok = F.check_iso(chi, p, h, lo, N, iso32(chi, p, h, lo, N))
    assert ok.ok, ok.describe()


def test_defect_rint_as_floor_half():
    p, _, ties = F.tie_cloud(6)
    g = O.grid(p, 6)
    N, h, lo = g["N"], g["h"], _lo(g)
    assert h == 2.0 ** -5
    rep, _ = F.check_cell_keys(p, None, h, lo, N, cell_keys32(p, h, lo, N))
    assert rep.ok, rep.describe()
    rep, _ = F.check_cell_keys(p, None, h, lo, N, cell_keys32(p, h, lo, N, "floor_half"))
    assert not rep.ok, rep.describe()
    i = rep.first_bad[0]
    q = p[i] / np.float32(h)
    assert ties[i] and (np.abs(q - np.floor(q)) == 0.5).any(), rep.describe()


def _normals_case():
    """Sphere cells plus an exactly collinear block and a 3-point block."""
    p, _ = O.sphere(20_000, seed=3, noise=0.001)
    line = np.stack([np.linspace(1.3, 1.4, 50), np.full(50, 1.3), np.full(50, 1.3)], 1)
    three = np.array([[-1.3, -1.3, -1.3], [-1.31, -1.3, -1.29], [-1.3, -1.31, -1.3]])
    p = np.concatenate([p, line, three]).astype(np.float32)
    g = O.grid(p, 6)
    N = g["N"]
    key = O.flat(O.cell_index(p, g), N)
    order = np.argsort(key, kind="stable")
    ps, ks = p[order], key[order]
    cells, start, cnt = np.unique(ks, return_index=True, return_counts=True)
    start = np.append(start, len(ks)).astype(np.int32)
    d = ps.astype(np.float64) - g["centre"]
    x, y, z = d.T
    t = np.stack([np.ones_like(x), x, y, z, x * x, x * y, x * z, y * y, y * z, z * z], 1)
    mom = np.add.reduceat(t, start[:-1], axis=0)
    return ps, g, cells, start, cnt, mom


def test_defect_eigenvector_column_order():
    ps, g, cells, start, cnt, mom = _normals_case()
    N = g["N"]
    assert F.check_moments(ps, start, g["centre"], mom).ok
    cn, cok = normals32(cells, mom, N)
    rep = F.check_normals(cells, mom, N, cn, cok)
    assert rep.ok and rep.exempt <= len(cells) // 100, rep.describe()
    assert not cok.all()                                        # the line and 3-point blocks
    cn_bad, _ = normals32(cells, mom, N, "eig_order")
    rep = F.check_normals(cells, mom, N, cn_bad, cok)
    assert not rep.ok, rep.describe()


def test_defect_camera_tie_to_the_higher_index():
    rng = np.random.default_rng(0)
    p = np.concatenate([rng.uniform(-1, 1, (3000, 2)), np.zeros((3000, 1))], 1).astype(np.float32)
    cams = np.array([[0, 0, 3.0], [0, 0, -3.0]])                  # every point equidistant
    cn = torch.tensor([[0.0, 0.0, 1.0], [0.0, 0.6, -0.8]], dtype=torch.float64)
    pcell = torch.from_numpy((rng.random(3000) < 0.5).astype(np.int64))
    rep = F.check_orient(p, pcell, cn, cams, orient32(p, pcell, cn, cams))
    assert rep.ok, rep.describe()
    rep = F.check_orient(p, pcell, cn, cams, orient32(p, pcell, cn, cams, "tie_high"))
    assert not rep.ok and rep.first_bad[0] == 0, rep.describe()


def test_convergence_check_fails_a_component_that_only_slows_the_cycle():
    """Per cycle, the restatement's contraction stays within CONTRACTION of the float64 cycle's.
    Weights (1/8, 1/4, 1/8) on one axis halve every coarse correction: the solve still reaches
    the tolerance or the cycle cap, but each cycle contracts far less, and the per-element
    restrict check fails it too.  (The (1/3, 1/3, 1/3) weights keep the sum 1 and barely change
    the contraction; only the per-element check sees them.)"""
    g, b, _ = _fields(6)
    _, want = F.multigrid64(b, g["h"])
    _, got = multigrid32(b, g["h"])
    assert F.contraction_ok(got, want), (got, want)
    _, bad = multigrid32(b, g["h"], "restrict_half")
    assert not F.contraction_ok(bad, want), (bad, want, F.CONTRACTION)
