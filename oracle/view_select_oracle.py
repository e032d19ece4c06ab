"""Float64 numpy restatement of the COLMAP scene conversion (casmvsnet_pl_b200/colmap.py and
csrc/view_select.cu): view-selection scores, source ranking, the reference-view skip rule and
the depth range.

    s(i,j)  = sum over points p with i, j in track(p) of G(theta_ij(p)), in ascending point order
    theta   = degrees(arccos(clip(dot(unit(c_i - p), unit(c_j - p)), -1, 1)))
    G       = exp(-(theta - 5)^2 / 2) if theta <= 5 else exp(-(theta - 5)^2 / 200)

view_scores loops over the points in order (the definition); view_scores_vec expands every pair
at once and adds them with np.add.at, which applies them in the same order."""
import numpy as np

THETA0, SIGMA1, SIGMA2 = 5.0, 1.0, 10.0


def weight(theta):
    theta = np.asarray(theta, np.float64)
    s = np.where(theta <= THETA0, SIGMA1, SIGMA2)
    return np.exp(-(theta - THETA0) ** 2 / (2 * s * s))


def _angle_weight(ci, cj, p):
    a, b = ci - p, cj - p
    na, nb = np.linalg.norm(a, axis=-1), np.linalg.norm(b, axis=-1)
    ok = (na > 0) & (nb > 0)
    na, nb = np.where(ok, na, 1), np.where(ok, nb, 1)
    dot = ((a / na[..., None]) * (b / nb[..., None])).sum(-1)
    return np.where(ok, weight(np.degrees(np.arccos(np.clip(dot, -1, 1)))), 0.0)


def view_scores(centres, xyz, track_ptr, track_img, n_img):
    """(n_img, n_img) float64, one point at a time in ascending order."""
    c = np.asarray(centres, np.float64)
    s = np.zeros((n_img, n_img))
    for p in range(len(xyz)):
        tr = [int(v) for v in track_img[track_ptr[p]:track_ptr[p + 1]]]
        for a in range(len(tr)):
            for b in range(a + 1, len(tr)):
                i, j = min(tr[a], tr[b]), max(tr[a], tr[b])
                if i == j or i < 0 or j >= n_img:
                    continue
                g = float(_angle_weight(c[i], c[j], np.asarray(xyz[p], np.float64)))
                s[i, j] += g
                s[j, i] = s[i, j]
    return s


def pair_entries(track_ptr, track_img):
    """Every pair of every track in the kernel's order: (point, i, j) arrays."""
    ptr = np.asarray(track_ptr, np.int64)
    img = np.asarray(track_img, np.int64)
    t = np.diff(ptr)
    pts, ii, jj = [], [], []
    for L in np.unique(t[t > 1]):
        sel = np.nonzero(t == L)[0]
        a, b = np.triu_indices(L, 1)
        base = ptr[sel][:, None]
        pts.append(np.repeat(sel, len(a)).reshape(len(sel), -1))
        ii.append(img[base + a])
        jj.append(img[base + b])
    if not pts:
        z = np.zeros(0, np.int64)
        return z, z, z
    p = np.concatenate([x.ravel() for x in pts])
    i = np.concatenate([x.ravel() for x in ii])
    j = np.concatenate([x.ravel() for x in jj])
    o = np.argsort(p, kind="stable")
    return p[o], i[o], j[o]


def view_scores_vec(centres, xyz, track_ptr, track_img, n_img):
    """view_scores with the pairs expanded at once (np.add.at adds in pair order)."""
    c = np.asarray(centres, np.float64)
    P = np.asarray(xyz, np.float64)
    p, i, j = pair_entries(track_ptr, track_img)
    lo, hi = np.minimum(i, j), np.maximum(i, j)
    ok = (lo != hi) & (lo >= 0) & (hi < n_img)
    p, lo, hi = p[ok], lo[ok], hi[ok]
    g = _angle_weight(c[lo], c[hi], P[p])
    s = np.zeros(n_img * n_img)
    np.add.at(s, lo * n_img + hi, g)
    s = s.reshape(n_img, n_img)
    return s + s.T


def select_sources(scores, n_src=10):
    """[[src]] per view: the n_src views with the highest positive score, ties to the lower id."""
    out = []
    for v, row in enumerate(np.asarray(scores)):
        cand = [(-row[j], j) for j in range(len(row)) if j != v and row[j] > 0]
        out.append([j for _, j in sorted(cand)[:n_src]])
    return out


def depth_range(E, xyz, track_ptr, track_img, v):
    """(count of z > 0, depth_min = 0.75 q(0.01), depth_max = 1.25 q(0.99)) of view v."""
    E = np.asarray(E, np.float64)
    zs = []
    for p in range(len(xyz)):
        if v in set(int(x) for x in track_img[track_ptr[p]:track_ptr[p + 1]]):
            z = E[v, 2, :3] @ np.asarray(xyz[p], np.float64) + E[v, 2, 3]
            if z > 0:
                zs.append(z)
    zs = np.sort(np.array(zs))
    n = len(zs)
    if n == 0:
        return 0, np.nan, np.nan
    q = lambda f: zs[int(np.floor(f * (n - 1)))]     # noqa: E731
    return n, 0.75 * q(0.01), 1.25 * q(0.99)


def skipped(n_sources, n_front, n_views, min_front=20):
    """True when a view cannot be a reference view."""
    return n_sources < n_views - 1 or n_front < min_front
