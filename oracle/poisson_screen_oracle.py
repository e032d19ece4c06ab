"""numpy float64 restatement of screened Poisson (poisson.py with point_weight > 0; the
casmvs_poisson_screen_* kernels of csrc/poisson.cu), built on oracle/poisson_oracle.py:

1. the unscreened solve gives chi0 and the target t = iso(chi0);
2. at interior nodes of level 0, L chi - gamma S chi = b - gamma t Phi, gamma = alpha (n_s / n) / h^2,
   S_ij = sum_p phi_i(p) phi_j(p), Phi_i = sum_p phi_i(p), n_s the number of splat cells;
3. per splat cell (floor corner), the 27 moments sum F_x^a F_y^b F_z^c;
4. level l uses L_l - (gamma / 8^l) S_l, its moments coarsened from the children under
   F' = (m + F) / 2;
5. 8-colour Gauss-Seidel V(2,2) cycles, 50 sweeps on the 8^3 level;
6. from chi0 until ||r|| / ||b_s|| <= 1e-5 or 40 cycles;
7. the iso level of the screened chi, then trim, colour, bricks and marching cubes unchanged.

Arrays follow poisson_oracle: level 0 is (N,N,N), a coarse level of n nodes is stored with
n + 1 entries per axis, entry n the Dirichlet node.  Never imported by the product."""
from __future__ import annotations

import numpy as np
from scipy import sparse
from scipy.sparse import linalg as splinalg

from oracle import mesh_oracle
from oracle import poisson_oracle as O

KEY_NONE = np.iinfo(np.int64).max
CORNERS = O.CORNERS                       # d = 4 dx + 2 dy + dz, x-major


def pair_coef(d, e):
    """Coefficients of 1, F, F^2 in w(d) w(e), w(0) = 1 - F, w(1) = F."""
    if d != e:
        return np.array([0.0, 1.0, -1.0])
    return np.array([0.0, 0.0, 1.0]) if d else np.array([1.0, -2.0, 1.0])


def single_coef(d):
    """Coefficients of 1, F, F^2 in w(d)."""
    return np.array([0.0, 1.0, 0.0]) if d else np.array([1.0, -1.0, 0.0])


def half_coef(m):
    """T[k', k]: coefficient of F^k in ((m + F) / 2)^k'."""
    return np.array([[1.0, 0, 0], [0.5, 0.5, 0], [0.25, 0.5, 0.25]]) if m else \
        np.diag([1.0, 0.5, 0.25])


def _powers(F):
    """(n,3) fractions -> (n,27) F_x^a F_y^b F_z^c, index 9a + 3b + c."""
    pw = [np.stack([np.ones(len(F)), F[:, a], F[:, a] * F[:, a]], 1) for a in range(3)]
    return ((pw[0][:, :, None, None] * pw[1][:, None, :, None]) * pw[2][:, None, None, :]).reshape(-1, 27)


def splat_keys(p, g):
    """Flat splat cell floor(p / h) - lo of each point on level 0, KEY_NONE when it leaves
    0..N-2 on an axis -> (keys (n,) int64, base (n,3) int64, frac (n,3) float32)."""
    base, frac = O._corners(p, g)
    N = g["N"]
    ok = ((base >= 0) & (base <= N - 2)).all(1)
    return np.where(ok, O.flat(np.where(ok[:, None], base, 0), N), KEY_NONE), base, frac


def moments(p, g, level=0):
    """Moments of every splat cell of level `level`, computed from the points: level l's cell is
    base >> l and its fraction ((base mod 2^l) + F) / 2^l (exact in double) -> (sorted flat cell
    keys on the (N >> l)^3 grid, M (cells, 27))."""
    key, base, frac = splat_keys(p, g)
    ok = key != KEY_NONE
    base, frac = base[ok], frac[ok].astype(np.float64)
    s = 1 << level
    n = g["N"] >> level
    F = ((base & (s - 1)) + frac) / s
    k = O.flat(base >> level, n)
    cells, inv = np.unique(k, return_inverse=True)
    M = np.zeros((len(cells), 27))
    np.add.at(M, inv, _powers(F))
    return cells, M


def coarsen(keys, M, n_child):
    """Parent cells of the (n_child/2)^3 grid and their moments, each the sum over its children of
    the child moments under F' = (m + F) / 2."""
    n = n_child // 2
    x, y, z = keys // (n_child * n_child), (keys // n_child) % n_child, keys % n_child
    pk = O.flat(np.stack([x >> 1, y >> 1, z >> 1], 1), n)
    out_keys, inv = np.unique(pk, return_inverse=True)
    T = [half_coef(0), half_coef(1)]
    Mc = M.reshape(-1, 3, 3, 3)
    moved = np.empty_like(Mc)
    for m in range(8):
        sel = ((x & 1) * 4 + (y & 1) * 2 + (z & 1)) == m
        moved[sel] = np.einsum("ia,jb,kc,nabc->nijk", T[m >> 2], T[(m >> 1) & 1], T[m & 1], Mc[sel])
    Mp = np.zeros((len(out_keys), 27))
    np.add.at(Mp, inv, moved.reshape(-1, 27))
    return out_keys, Mp


def level_moments(p, g):
    """[(keys, M)] of level 0 from the points and of every coarser level down to 8^3 by coarsen."""
    out = [moments(p, g, 0)]
    n = g["N"]
    while n // 2 >= O.COARSEST:
        out.append(coarsen(*out[-1], n))
        n //= 2
    return out


def _pair_table():
    C = np.zeros((8, 8, 27))
    for d, (dx, dy, dz) in enumerate(CORNERS):
        for e, (ex, ey, ez) in enumerate(CORNERS):
            C[d, e] = np.einsum("a,b,c->abc", pair_coef(dx, ex), pair_coef(dy, ey),
                                pair_coef(dz, ez)).ravel()
    return C


def _phi_table():
    return np.stack([np.einsum("a,b,c->abc", single_coef(dx), single_coef(dy), single_coef(dz)).ravel()
                     for dx, dy, dz in CORNERS])


def cell_blocks(M):
    """-> (S (cells,8,8) = sum phi_d phi_e, Phi (cells,8) = sum phi_d) from the moments."""
    return np.einsum("nk,dek->nde", M, _pair_table()), M @ _phi_table().T


def screen_matrix(keys, M, n, m):
    """S (m^3 x m^3 scipy.sparse, the array layout of m entries per axis) and Phi (m,m,m) of a
    level of n stored nodes per axis: corners at index n (a coarse level's unstored Dirichlet
    node) drop."""
    x, y, z = keys // (n * n), (keys // n) % n, keys % n
    S, Phi = cell_blocks(M)
    rows, cols, vals = [], [], []
    phi = np.zeros(m ** 3)
    for d, (dx, dy, dz) in enumerate(CORNERS):
        okd = (x + dx < n) & (y + dy < n) & (z + dz < n)
        i = ((x + dx) * m + (y + dy)) * m + (z + dz)
        np.add.at(phi, i[okd], Phi[okd, d])
        for e, (ex, ey, ez) in enumerate(CORNERS):
            ok = okd & (x + ex < n) & (y + ey < n) & (z + ez < n)
            j = ((x + ex) * m + (y + ey)) * m + (z + ez)
            rows.append(i[ok])
            cols.append(j[ok])
            vals.append(S[ok, d, e])
    A = sparse.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))),
                          shape=(m ** 3, m ** 3)).tocsr()
    return A, phi.reshape(m, m, m)


def prolongation(nc):
    """P: coarse ((nc + 1)^3 layout, entry nc the Dirichlet node) -> fine ((2 nc)^3), trilinear,
    as O.prolong, for the Galerkin identity P^T S_f P = S_c."""
    def one(nf):
        rows, cols, vals = [], [], []
        for i in range(nf):
            if i % 2 == 0:
                rows.append(i), cols.append(i // 2), vals.append(1.0)
            else:
                for c in (i // 2, i // 2 + 1):
                    rows.append(i), cols.append(c), vals.append(0.5)
        return sparse.coo_matrix((vals, (rows, cols)), shape=(nf, nc + 1)).tocsr()
    p1 = one(2 * nc)
    return sparse.kron(sparse.kron(p1, p1), p1).tocsr()


def level_ops(levels, g, gg):
    """[(S_l in the level's array layout, g_l = gg / 2^l)] for the multigrid."""
    N = g["N"]
    ops = []
    for l, (keys, M) in enumerate(levels):
        n = N >> l
        S, _ = screen_matrix(keys, M, n, n if l == 0 else n + 1)
        ops.append((S, gg / 2 ** l))
    return ops


def apply_screened(x, h, S, gl):
    """(nbsum - 6 x - gl S x) / h^2 at interior nodes, 0 elsewhere."""
    Sx = (S @ x.reshape(-1)).reshape(x.shape)
    return np.where(O._interior(len(x)), (O._nbsum(x) - 6 * x - gl * Sx) / (h * h), 0.0)


def colour_of(m):
    x, y, z = np.indices((m, m, m))
    return 4 * (x & 1) + 2 * (y & 1) + (z & 1)


def smooth(e, r, h, S, gl, sweeps):
    """`sweeps` 8-colour Gauss-Seidel sweeps, colours 0..7 in order."""
    m = len(e)
    inner = O._interior(m)
    col = colour_of(m)
    diag = S.diagonal().reshape(e.shape)
    for _ in range(sweeps):
        for k in range(8):
            sel = inner & (col == k)
            off = (S @ e.reshape(-1)).reshape(e.shape) - diag * e
            new = (O._nbsum(e) - h * h * r - gl * off) / (6 + gl * diag)
            e[sel] = new[sel]
    return e


def vcycle(r, h, ops, l=0, pre=2, post=2, coarse_sweeps=50):
    """One screened V(pre, post) cycle for A_l e = r from e = 0 (as O.vcycle)."""
    S, gl = ops[l]
    m = len(r)
    e = np.zeros_like(r)
    if m - m % 2 <= O.COARSEST:
        return smooth(e, r, h, S, gl, coarse_sweeps)
    smooth(e, r, h, S, gl, pre)
    res = np.where(O._interior(m), r - apply_screened(e, h, S, gl), 0.0)
    ec = vcycle(O.restrict(res), 2 * h, ops, l + 1, pre, post, coarse_sweeps)
    e += np.where(O._interior(m), O.prolong(ec, m), 0.0)
    return smooth(e, r, h, S, gl, post)


def multigrid(b_s, chi0, h, ops, tol=1e-5, max_cycles=40):
    """From chi0, V(2,2) cycles until ||r|| / ||b_s|| <= tol or max_cycles -> (chi, cycles,
    ratios before each cycle and at the end)."""
    chi = chi0.copy()
    bn = O.norm2(b_s)
    if bn == 0:
        return chi, 0, [0.0]
    S, g0 = ops[0]
    cycles, ratios = 0, []
    while True:
        r = np.where(O._interior(len(b_s)), b_s - apply_screened(chi, h, S, g0), 0.0)
        ratios.append(O.norm2(r) / bn)
        if ratios[-1] <= tol or cycles == max_cycles:
            return chi, cycles, ratios
        chi += vcycle(r, h, ops)
        cycles += 1


def direct_solve(b_s, h, S, gg):
    """L chi - (gg / h^2) S chi = b_s at interior nodes (chi = 0 on the outer layer) by spsolve."""
    n = len(b_s)
    m = n - 2
    one = sparse.identity(m, format="csr")
    t = sparse.diags([np.ones(m - 1), -2 * np.ones(m), np.ones(m - 1)], [-1, 0, 1], format="csr")
    L = (sparse.kron(sparse.kron(t, one), one) + sparse.kron(sparse.kron(one, t), one)
         + sparse.kron(sparse.kron(one, one), t)) / (h * h)
    inner = np.flatnonzero(O._interior(n).reshape(-1))
    A = L - (gg / (h * h)) * S[inner][:, inner]
    chi = np.zeros_like(b_s)
    chi[1:-1, 1:-1, 1:-1] = splinalg.spsolve(A.tocsc(), b_s[1:-1, 1:-1, 1:-1].reshape(-1)).reshape(m, m, m)
    return chi


def screened_system(pk, g, b, t, alpha):
    """-> dict(levels, n_s, g (alpha n_s / n), gamma, S0, Phi, b_s, ops) of the kept points pk."""
    levels = level_moments(pk, g)
    N, h = g["N"], g["h"]
    n_s = len(levels[0][0])
    gg = alpha * n_s / len(pk)
    gamma = gg / (h * h)
    S0, Phi = screen_matrix(*levels[0], N, N)
    b_s = np.where(O._interior(N), b - gamma * t * Phi, 0.0)
    return dict(levels=levels, n_s=n_s, g=gg, gamma=gamma, S0=S0, Phi=Phi, b_s=b_s,
                ops=level_ops(levels, g, gg))


def poisson(xyz, rgb=None, normals=None, cams=None, depth=9, point_weight=0.0, tol=1e-5,
            max_cycles=40):
    """poisson_oracle.poisson with the point-weight term -> its dict with chi, iso and the mesh of
    the screened field, plus chi0, target, b_s, levels, g, screened_cycles, screened_ratios."""
    r = O.poisson(xyz, rgb, normals, cams, depth, tol, max_cycles)
    g, pk = r["grid"], r["points"]
    sys_ = screened_system(pk, g, r["b"], r["iso"], point_weight)
    chi, cycles, ratios = multigrid(sys_["b_s"], r["chi"], g["h"], sys_["ops"], tol, max_cycles)
    iso = O.iso_level(chi, pk, g)
    f = chi - iso
    keys, tsdf, weight, color = O.bricks(f, r["keep"], r["colour"], g)
    verts, colours, faces = mesh_oracle.extract(keys, tsdf, weight, color, g["h"])
    out = dict(r, chi0=r["chi"], target=r["iso"], chi=chi, iso=iso, keys=keys, tsdf=tsdf,
               weight=weight, color=color, verts=verts, colours=colours, faces=faces,
               screened_cycles=cycles, screened_ratios=ratios)
    out.update({k: sys_[k] for k in ("levels", "n_s", "g", "gamma", "b_s")})
    return out


# ------------------------------------------------------------------------------ test clouds
def cube(n, side=1.0, seed=0, noise=0.0):
    """n points uniform on the six faces of an axis-aligned cube of side `side` centred at the
    origin, rotated by a seeded rotation, with exact outward normals -> (xyz, normals) float32 and
    the rotation q (world = cube @ q)."""
    rng = np.random.default_rng(seed)
    face = rng.integers(0, 6, n)
    uv = rng.uniform(-side / 2, side / 2, (n, 2))
    ax = face // 2
    sgn = np.where(face % 2 == 0, 1.0, -1.0)
    p = np.empty((n, 3))
    nrm = np.zeros((n, 3))
    for a in range(3):
        sel = ax == a
        o = [b for b in range(3) if b != a]
        p[sel, a] = sgn[sel] * side / 2 + noise * rng.normal(size=sel.sum())
        p[sel, o[0]], p[sel, o[1]] = uv[sel, 0], uv[sel, 1]
        nrm[sel, a] = sgn[sel]
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return (p @ q).astype(np.float32), (nrm @ q).astype(np.float32), q


def cube_distance(v, q, side=1.0):
    """Distance of points v (world) from the surface of the cube rotated by q."""
    u = np.abs(np.asarray(v, np.float64) @ q.T) - side / 2       # back to the cube's axes
    outside = np.linalg.norm(np.maximum(u, 0), axis=1)
    inside = np.minimum(u.max(1), 0)
    return np.abs(outside + inside)


# ------------------------------------------------------------------------------ per-node rows
def stencil_rows(nodes, keys, M, n):
    """27-point stencils of S (k = 9 (dx+1) + 3 (dy+1) + (dz+1)) at nodes (K,3) of a level of n
    stored nodes, from the moments of its sorted cells; corners at index n drop -> (K,27), and
    Phi at the nodes (K,)."""
    nodes = np.asarray(nodes, np.int64)
    table, ptab = _pair_table(), _phi_table()
    rows, phi = np.zeros((len(nodes), 27)), np.zeros(len(nodes))
    for d, (dx, dy, dz) in enumerate(CORNERS):
        c = nodes - np.array([dx, dy, dz])
        key = O.flat(np.maximum(c, 0), n)
        pos = np.minimum(np.searchsorted(keys, key), max(len(keys) - 1, 0))
        hit = (c >= 0).all(1) & (len(keys) > 0) & (keys[pos] == key)
        if not hit.any():
            continue
        Mh = M[pos[hit]]
        phi[hit] += Mh @ ptab[d]
        S = Mh @ table[d].T                                      # (h, 8): corners t of the cell
        for t, (tx, ty, tz) in enumerate(CORNERS):
            ok = ((c[hit] + np.array([tx, ty, tz])) < n).all(1)
            k = (tx - dx + 1) * 9 + (ty - dy + 1) * 3 + (tz - dz + 1)
            idx = np.flatnonzero(hit)[ok]
            rows[idx, k] += S[ok, t]
    return rows, phi


OFFSETS = np.array([(k // 9 - 1, (k // 3) % 3 - 1, k % 3 - 1) for k in range(27)])


def window_sweep(E, R, origin, n, level, h, gl, rows, colours=range(8)):
    """One 8-colour sweep on a box E (float64, global origin `origin`) of a level, rows the (box
    nodes, 27) stencils of S in the box's C order.  Nodes on the box's border are not updated, so
    only nodes 8 or more from the border are exact."""
    E = E.copy()
    b = np.array(E.shape)
    g = np.indices(E.shape).reshape(3, -1).T + np.asarray(origin)
    top = n if level else n - 1
    inner_g = ((g > 0) & (g < top)).all(1)
    loc = np.indices(E.shape).reshape(3, -1).T
    inner_b = ((loc > 0) & (loc < b - 1)).all(1)
    col = 4 * (g[:, 0] & 1) + 2 * (g[:, 1] & 1) + (g[:, 2] & 1)
    flatE = E.reshape(-1)
    R = R.reshape(-1)
    strides = np.array([b[1] * b[2], b[2], 1])
    for k in colours:
        sel = np.flatnonzero(inner_g & inner_b & (col == k))
        nb = np.zeros(len(sel))
        off = np.zeros(len(sel))
        for j, o in enumerate(OFFSETS):
            if j == 13:
                continue
            v = flatE[sel + o @ strides]
            if abs(o).sum() == 1:
                nb += v
            off += rows[sel, j] * v
        flatE[sel] = (nb - h * h * R[sel] - gl * off) / (6 + gl * rows[sel, 13])
    return E
