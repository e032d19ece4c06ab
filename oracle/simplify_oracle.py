"""numpy float64 restatement of quadric edge-collapse decimation (simplify.py; the
casmvs_simplify_* kernels of csrc/simplify.cu), round by round, bit for bit, plus a serial greedy
QEM (one cheapest valid collapse at a time) with the same quadrics and validity, used only to
judge fidelity.

Every double operation is rounded to nearest in the order written below (numpy does not
contract), as the kernels do with __dmul_rn / __dadd_rn.  Sums over several items use np.add.at,
which applies its items in index order.  Never imported by the product."""
from __future__ import annotations

import heapq
import math

import numpy as np
from scipy import sparse

MAX_FAN = 32
BOUNDARY_WEIGHT = 1000.0
CANDIDATE_DIVISOR = 4            # candidates: keys <= the ceil(E_valid / 4)-th smallest valid key
FOLD_COS = 0.2
DET_EPS = 1e-12
KEY_NONE = np.iinfo(np.int64).max
# the 10 unique entries of a symmetric 4x4 quadric, row-major upper triangle
QIDX = ((0, 0), (0, 1), (0, 2), (0, 3), (1, 1), (1, 2), (1, 3), (2, 2), (2, 3), (3, 3))
f32, f64 = np.float32, np.float64


# ------------------------------------------------------------------------------ geometry
def cross(u, v):
    return np.stack([u[..., 1] * v[..., 2] - u[..., 2] * v[..., 1],
                     u[..., 2] * v[..., 0] - u[..., 0] * v[..., 2],
                     u[..., 0] * v[..., 1] - u[..., 1] * v[..., 0]], -1)


def dot(u, v):
    return (u[..., 0] * v[..., 0] + u[..., 1] * v[..., 1]) + u[..., 2] * v[..., 2]


def face_normals(P, faces):
    """Unnormalised n = (p1 - p0) x (p2 - p0) in double, P (V,3) float32."""
    p = P.astype(f64)[faces]
    return cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])


def plane_quadric(nrm, p0, w):
    """w * [n^, -n^.p0][n^, -n^.p0]^T (10 unique entries), n^ = nrm / |nrm|."""
    ln = np.sqrt(dot(nrm, nrm))
    nh = nrm / ln[..., None]
    pl = np.concatenate([nh, -dot(nh, p0)[..., None]], -1)
    return np.stack([w * (pl[..., i] * pl[..., j]) for i, j in QIDX], -1)


def clean(P, faces):
    """-> keep flags: faces without a repeated index and with n != 0 in double."""
    f = faces.astype(np.int64)
    rep = (f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) | (f[:, 0] == f[:, 2])
    n = face_normals(P, f)
    return ~rep & ~(n == 0).all(1)


# ------------------------------------------------------------------------------ topology
def edges(faces):
    """-> (edge keys (E,) sorted, a, b, corner -> edge (3F,), faces per edge (E,)).  Corner
    c = 3 f + k owns the edge faces[f,k] -- faces[f,(k+1)%3]."""
    f = faces.astype(np.int64)
    g = np.roll(f, -1, axis=1)
    key = (np.minimum(f, g) << 32) | np.maximum(f, g)
    ek, inv, cnt = np.unique(key.ravel(), return_inverse=True, return_counts=True)
    return ek, ek >> 32, ek & 0xFFFFFFFF, inv.ravel(), cnt


def csr(faces, V):
    """vertex -> corners (3 f + k) in face order: (offsets (V+1,), corners)."""
    flat = faces.astype(np.int64).ravel()
    order = np.argsort(flat, kind="stable")
    off = np.concatenate([[0], np.cumsum(np.bincount(flat, minlength=V))])
    return off, order


def frozen_flags(faces, V):
    """Vertices on an edge of > 2 faces, with > MAX_FAN faces, or whose faces do not form one
    fan (the link graph, an edge (p, q) per face (v, p, q), is not connected)."""
    ek, a, b, inv, cnt = edges(faces)
    nfan = np.bincount(faces.ravel(), minlength=V)
    frozen = nfan > MAX_FAN
    frozen[a[cnt > 2]] = True
    frozen[b[cnt > 2]] = True
    off, order = csr(faces, V)
    for v in np.nonzero((nfan > 0) & ~frozen)[0]:
        fs = faces[order[off[v]:off[v + 1]] // 3]
        link = [tuple(int(x) for x in f if x != v) for f in fs]
        seen, stack = {link[0][0]}, [link[0][0]]
        while stack:
            x = stack.pop()
            for p, q in link:
                for s, t in ((p, q), (q, p)):
                    if s == x and t not in seen:
                        seen.add(t)
                        stack.append(t)
        if len(seen) != len({x for pq in link for x in pq}):
            frozen[v] = True
    return frozen


# ------------------------------------------------------------------------------ quadrics
def vertex_quadrics(P, faces, V):
    """Q_v (V,10): incident face quadrics in face order, then boundary-edge quadrics in key
    order."""
    n = face_normals(P, faces)
    p0 = P.astype(f64)[faces[:, 0]]
    fq = plane_quadric(n, p0, np.sqrt(dot(n, n)) * 0.5)
    Q = np.zeros((V, 10))
    np.add.at(Q, faces.astype(np.int64).ravel(), np.repeat(fq, 3, axis=0))
    ek, a, b, inv, cnt = edges(faces)
    bd = np.nonzero(cnt == 1)[0]
    if len(bd):
        face_of = np.zeros(len(ek), np.int64)
        face_of[inv] = np.arange(len(inv)) // 3
        pa, pb = P.astype(f64)[a[bd]], P.astype(f64)[b[bd]]
        e = pb - pa
        bq = plane_quadric(cross(e, n[face_of[bd]]), pa, BOUNDARY_WEIGHT * dot(e, e))
        ends = np.stack([a[bd], b[bd]], 1).ravel()
        np.add.at(Q, ends, np.repeat(bq, 2, axis=0))
    return Q


def qform(q, x):
    """[x,1]^T Q [x,1] in double, x (...,3)."""
    x0, x1, x2 = x[..., 0], x[..., 1], x[..., 2]
    u0 = ((q[..., 0] * x0 + q[..., 1] * x1) + q[..., 2] * x2) + q[..., 3]
    u1 = ((q[..., 1] * x0 + q[..., 4] * x1) + q[..., 5] * x2) + q[..., 6]
    u2 = ((q[..., 2] * x0 + q[..., 5] * x1) + q[..., 7] * x2) + q[..., 8]
    u3 = ((q[..., 3] * x0 + q[..., 6] * x1) + q[..., 8] * x2) + q[..., 9]
    return ((u0 * x0 + u1 * x1) + u2 * x2) + u3


def det3(m00, m01, m02, m10, m11, m12, m20, m21, m22):
    return ((m00 * (m11 * m22 - m12 * m21) - m01 * (m10 * m22 - m12 * m20))
            + m02 * (m10 * m21 - m11 * m20))


def position_cost(q, pa, pb):
    """Per edge, Q = Q_a + Q_b (E,10), endpoints float32 -> (v (E,3) float32, cost (E,) float32
    or NaN).  Cramer's rule when |det A| > DET_EPS max|A_ij|^3 and the rounded v is finite,
    else the first cheapest of a, b, midpoint."""
    a00, a01, a02, a11, a12, a22 = (q[:, i] for i in (0, 1, 2, 4, 5, 7))
    r0, r1, r2 = -q[:, 3], -q[:, 6], -q[:, 8]
    det = det3(a00, a01, a02, a01, a11, a12, a02, a12, a22)
    m = np.max(np.abs(np.stack([a00, a01, a02, a11, a12, a22], 1)), 1)
    with np.errstate(all="ignore"):
        x = np.stack([det3(r0, a01, a02, r1, a11, a12, r2, a12, a22) / det,
                      det3(a00, r0, a02, a01, r1, a12, a02, r2, a22) / det,
                      det3(a00, a01, r0, a01, a11, r1, a02, a12, r2) / det], 1).astype(f32)
        solve = (np.abs(det) > DET_EPS * ((m * m) * m)) & np.isfinite(x).all(1)
        pm = ((pa.astype(f64) + pb.astype(f64)) * 0.5).astype(f32)
        ca, cb, cm = (qform(q, p.astype(f64)) for p in (pa, pb, pm))
        fb = np.where(((ca <= cb) & (ca <= cm))[:, None], pa,
                      np.where((cb <= cm)[:, None], pb, pm))
        v = np.where(solve[:, None], x, fb).astype(f32)
        c = qform(q, v.astype(f64))
        cost = np.where(c > 0, c, 0.0).astype(f32)
        cost[np.isnan(c)] = np.nan
    return v, cost


# ------------------------------------------------------------------------------ one round
def round_state(P, Q, faces, frozen, max_error=None):
    """Edges, positions, costs, validity and keys of the current mesh."""
    V, F = len(P), len(faces)
    ek, a, b, inv, cnt = edges(faces)
    E = len(ek)
    off, order = csr(faces, V)
    deg = np.bincount(a, minlength=V) + np.bincount(b, minlength=V)
    bnd = np.zeros(V, bool)
    bnd[a[cnt == 1]] = bnd[b[cnt == 1]] = True
    nfan = np.bincount(faces.ravel(), minlength=V)
    v, cost = position_cost(Q[a] + Q[b], P[a], P[b])

    ok = ~frozen[a] & ~frozen[b] & np.isfinite(cost)
    adj = sparse.csr_matrix((np.ones(2 * E), (np.concatenate([a, b]), np.concatenate([b, a]))),
                            shape=(V, V))
    ncommon = np.asarray((adj @ adj)[a, b]).ravel().astype(np.int64)
    # opposite vertex of each corner's edge
    ff = faces.astype(np.int64)
    opp = np.roll(ff, -2, axis=1).ravel()
    s = np.argsort(inv, kind="stable")
    start = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    o1 = opp[s][start]
    o2 = opp[s][np.minimum(start + 1, 3 * F - 1)]
    ndist = 1 + ((cnt >= 2) & (o2 != o1))
    ok &= ncommon == ndist
    ok &= ~(bnd[a] & bnd[b]) | (cnt == 1)
    ok &= deg[a] + deg[b] - 2 - ncommon >= np.where(bnd[a] | bnd[b], 2, 3)
    opp_ok = deg[opp] - 1 >= np.where(bnd[opp], 2, 3)
    eo = np.ones(E, bool)
    np.logical_and.at(eo, inv, opp_ok)
    ok &= eo
    ok &= nfan[a] + nfan[b] - cnt <= MAX_FAN
    # folds: every face around a or b that does not hold both
    ed = np.nonzero(ok)[0]
    if len(ed):
        u = np.stack([a[ed], b[ed]], 1).ravel()
        eid = np.repeat(ed, 2)
        n_u = nfan[u]
        rep = np.repeat(np.arange(len(u)), n_u)
        pos = off[u][rep] + np.arange(n_u.sum()) - np.repeat(np.cumsum(n_u) - n_u, n_u)
        corner = order[pos]
        fi, k = corner // 3, corner % 3
        e = eid[rep]
        fv = ff[fi]
        both = ((fv == a[e][:, None]).any(1) & (fv == b[e][:, None]).any(1))
        p_old = P.astype(f64)[fv]
        p_new = p_old.copy()
        p_new[np.arange(len(fi)), k] = v[e].astype(f64)
        no = cross(p_old[:, 1] - p_old[:, 0], p_old[:, 2] - p_old[:, 0])
        nn = cross(p_new[:, 1] - p_new[:, 0], p_new[:, 2] - p_new[:, 0])
        good = dot(nn, no) > (FOLD_COS * np.sqrt(dot(nn, nn))) * np.sqrt(dot(no, no))
        fold_ok = np.ones(E, bool)
        np.logical_and.at(fold_ok, e, good | both)
        ok &= fold_ok
    valid0 = ok
    valid = valid0 & (True if max_error is None else cost.astype(f64) <= max_error)
    bits = cost.view(np.uint32).astype(np.int64)
    key = np.where(valid, (bits << 32) | np.arange(E, dtype=np.int64), KEY_NONE)
    return dict(ek=ek, a=a, b=b, cnt=cnt, v=v, cost=cost, valid0=valid0, valid=valid, key=key,
                deg=deg, bnd=bnd)


def select(st, faces, V):
    """Candidates, then the edges whose key is the least over the 1-rings of both endpoints."""
    key, a, b = st["key"], st["a"], st["b"]
    nv = int(st["valid"].sum())
    if nv == 0:
        return np.zeros(len(key), bool), None
    k = (nv + CANDIDATE_DIVISOR - 1) // CANDIDATE_DIVISOR
    thr = np.partition(key, k - 1)[k - 1]
    cand = key <= thr
    m1 = np.full(V, KEY_NONE, np.int64)
    np.minimum.at(m1, a[cand], key[cand])
    np.minimum.at(m1, b[cand], key[cand])
    m2 = m1.copy()
    fm = m1[faces].min(1)
    np.minimum.at(m2, faces.astype(np.int64).ravel(), np.repeat(fm, 3))
    return cand & (key == m2[a]) & (key == m2[b]), thr


def budget(st, sel, F, target):
    """Selected edges in key order, cut to the shortest prefix that removes >= F - target faces."""
    idx = np.nonzero(sel)[0]
    idx = idx[np.argsort(st["key"][idx], kind="stable")]
    removed = np.cumsum(st["cnt"][idx])
    n = min(len(idx), int(np.searchsorted(removed, F - target, "left")) + 1)
    return idx[:n]


def collapse(P, C, Q, faces, st, idx):
    """Apply the collapses `idx` in place on P, C, Q -> compacted faces."""
    a, b, v = st["a"][idx], st["b"][idx], st["v"][idx]
    pa, pb = P[a].astype(f64), P[b].astype(f64)
    e = pb - pa
    den = dot(e, e)
    with np.errstate(all="ignore"):
        t = np.where(den > 0, dot(v.astype(f64) - pa, e) / den, 0.0)
    t = np.minimum(np.maximum(t, 0.0), 1.0)
    ca, cb = C[a].astype(f64), C[b].astype(f64)
    C[a] = np.clip(np.rint(ca + t[:, None] * (cb - ca)), 0, 255).astype(np.uint8)
    Q[a] = Q[a] + Q[b]
    P[a] = v
    remap = np.arange(len(P), dtype=np.int64)
    remap[b] = a
    f = remap[faces]
    keep = (f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])
    return f[keep].astype(np.int32)


def prepare(verts, colours, faces):
    P = np.asarray(verts, f32).reshape(-1, 3).copy()
    C = np.asarray(colours, np.uint8).reshape(-1, 3).copy()
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    keep = clean(P, f)
    f = f[keep].astype(np.int32)
    frozen = frozen_flags(f, len(P))
    Q = vertex_quadrics(P, f, len(P))
    return P, C, f, frozen, Q, int((~keep).sum())


def compact(P, C, faces):
    used = np.zeros(len(P), bool)
    used[faces.ravel()] = True
    new = np.cumsum(used) - 1
    return P[used], C[used], new[faces].astype(np.int32)


def simplify(verts, colours, faces, target, max_error=None, trace=None):
    """The whole parallel decimation -> (verts, colours, faces, stats).  `trace`, a list,
    receives each round's state, selection and chosen edges."""
    P, C, f, frozen, Q, dropped = prepare(verts, colours, faces)
    F0, rounds, collapses, max_cost, stop = len(faces), 0, 0, 0.0, "target"
    while len(f) > target:
        st = round_state(P, Q, f, frozen, max_error)
        sel, thr = select(st, f, len(P))
        if thr is None:
            stop = "max_error" if max_error is not None and st["valid0"].any() else "no_candidate"
            break
        idx = budget(st, sel, len(f), target)
        if trace is not None:
            trace.append(dict(st, sel=sel, thr=thr, idx=idx, Q=Q.copy()))
        max_cost = max(max_cost, float(st["cost"][idx].max()))
        f = collapse(P, C, Q, f, st, idx)
        rounds += 1
        collapses += len(idx)
    V, Cc, F = compact(P, C, f)
    return V, Cc, F, dict(faces_in=F0, vertices_in=len(verts), faces=len(F), vertices=len(V),
                          rounds=rounds, collapses=collapses, max_cost=max_cost,
                          frozen_vertices=int(frozen.sum()), dropped_faces=dropped, stop=stop)


# ------------------------------------------------------------------------------ serial greedy
def serial_simplify(verts, colours, faces, target):
    """Greedy QEM: repeatedly collapse the cheapest valid edge (same quadrics, position rule and
    validity as above, checked on the current mesh) until <= target faces or none is valid."""
    P, C, f, frozen, Q, _ = prepare(verts, colours, faces)
    faces_l = [list(map(int, x)) for x in f]
    alive = [True] * len(faces_l)
    fan = [set() for _ in range(len(P))]
    for i, x in enumerate(faces_l):
        for u in x:
            fan[u].add(i)
    stamp = [0] * len(P)
    heap = []

    def nbrs(u):
        return {w for i in fan[u] for w in faces_l[i] if w != u}

    def is_bnd(u):
        return any(sum(w in faces_l[i] for i in fan[u]) == 1 for w in nbrs(u))

    def fold_ok(pts, k, v):
        def nrm(p):
            u = [p[1][i] - p[0][i] for i in range(3)]
            w = [p[2][i] - p[0][i] for i in range(3)]
            return (u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0])
        no = nrm(pts)
        pts = list(pts)
        pts[k] = v
        nn = nrm(pts)
        d = (nn[0] * no[0] + nn[1] * no[1]) + nn[2] * no[2]
        return d > (FOLD_COS * math.sqrt((nn[0] * nn[0] + nn[1] * nn[1]) + nn[2] * nn[2])) * \
            math.sqrt((no[0] * no[0] + no[1] * no[1]) + no[2] * no[2])

    def valid(a, b, v):
        if frozen[a] or frozen[b]:
            return False
        on = [i for i in fan[a] if b in faces_l[i]]
        na, nb_ = nbrs(a), nbrs(b)
        common = (na & nb_) - {a, b}
        opp = {w for i in on for w in faces_l[i] if w not in (a, b)}
        if common != opp:
            return False
        ba, bb = is_bnd(a), is_bnd(b)
        if ba and bb and len(on) != 1:
            return False
        if len(na) + len(nb_) - 2 - len(common) < (2 if ba or bb else 3):
            return False
        if any(len(nbrs(c)) - 1 < (2 if is_bnd(c) else 3) for c in opp):
            return False
        if len(fan[a]) + len(fan[b]) - len(on) > MAX_FAN:
            return False
        for u in (a, b):
            for i in fan[u]:
                x = faces_l[i]
                if a in x and b in x:
                    continue
                if not fold_ok([tuple(map(float, P[w])) for w in x], x.index(u), v):
                    return False
        return True

    def push(pairs):
        if not pairs:
            return
        ab = np.array(sorted({(min(p), max(p)) for p in pairs}), np.int64)
        v, c = position_cost(Q[ab[:, 0]] + Q[ab[:, 1]], P[ab[:, 0]], P[ab[:, 1]])
        for (a, b), vv, cc in zip(ab.tolist(), v.tolist(), c.tolist()):
            if math.isfinite(cc):
                heapq.heappush(heap, (cc, a, b, stamp[a], stamp[b], tuple(vv)))

    push([(a, w) for a in range(len(P)) for w in nbrs(a) if w > a])
    n_faces = len(faces_l)
    while n_faces > target and heap:
        c, a, b, sa, sb, v = heapq.heappop(heap)
        if sa != stamp[a] or sb != stamp[b] or not fan[a] or not fan[b]:
            continue
        if not valid(a, b, v):
            continue
        on = [i for i in fan[a] if b in faces_l[i]]
        for i in on:
            alive[i] = False
            for u in faces_l[i]:
                fan[u].discard(i)
        n_faces -= len(on)
        for i in fan[b]:
            faces_l[i] = [a if u == b else u for u in faces_l[i]]
            fan[a].add(i)
        fan[b] = set()
        Q[a] = Q[a] + Q[b]
        P[a] = v
        ring = nbrs(a)
        for u in ring | {a}:
            stamp[u] += 1
        push([(u, w) for u in ring | {a} for w in nbrs(u)])
    f = np.array([x for x, al in zip(faces_l, alive) if al], np.int32).reshape(-1, 3)
    return compact(P, C, f)


# ------------------------------------------------------------------------------ test meshes
def grid_mesh(n, size=1.0):
    """A flat (n+1)^2-vertex square grid in z = 0, 2 n^2 faces, counter-clockwise seen from +z."""
    t = np.linspace(0.0, size, n + 1)
    x, y = np.meshgrid(t, t, indexing="xy")
    verts = np.stack([x.ravel(), y.ravel(), np.zeros(x.size)], 1).astype(f32)
    i = np.arange(n)[None, :] + (n + 1) * np.arange(n)[:, None]
    i = i.ravel()
    faces = np.concatenate([np.stack([i, i + 1, i + n + 2], 1), np.stack([i, i + n + 2, i + n + 1], 1)])
    return verts, faces.astype(np.int32)


def cube_mesh(n, side=1.0):
    """A closed cube of `side` centred at the origin, n x n quads (2 triangles each) per face,
    shared vertices, outward winding."""
    idx = {}
    verts, faces = [], []

    def vid(p):
        k = tuple(int(c) for c in p)
        if k not in idx:
            idx[k] = len(verts)
            verts.append(k)
        return idx[k]
    for axis in range(3):
        for sgn in (0, n):
            u, w = [d for d in range(3) if d != axis]
            for i in range(n):
                for j in range(n):
                    q = []
                    for di, dj in ((0, 0), (1, 0), (1, 1), (0, 1)):
                        p = [0, 0, 0]
                        p[axis], p[u], p[w] = sgn, i + di, j + dj
                        q.append(vid(p))
                    faces.append([q[0], q[1], q[2]])
                    faces.append([q[0], q[2], q[3]])
    V = np.array(verts, f64) / n * side - side / 2
    F = np.array(faces, np.int64)
    # orient outward: flip faces whose normal points towards the centre
    p = V[F]
    nrm = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    flip = np.einsum("ij,ij->i", nrm, p.mean(1)) < 0
    F[flip] = F[flip][:, ::-1]
    return V.astype(f32), F.astype(np.int32)


def sphere_mesh(n, radius=1.0):
    """A closed marching-cubes sphere of `radius` at the origin from an n^3 analytic signed
    distance grid (oracle/mesh_oracle.py), outward winding; colours vary with position."""
    from oracle import mesh_oracle
    h = 2.6 * radius / n
    c = (np.arange(n) - (n - 1) / 2) * h
    x, y, z = np.meshgrid(c, c, c, indexing="ij")
    sdf = (np.sqrt(x * x + y * y + z * z) - radius) / h
    keys, tsdf, weight, color = mesh_oracle.grid_volume(sdf)
    color = np.zeros_like(color)
    color[:, 0] = np.tile(np.arange(512) % 8 * 32, len(keys))
    verts, cols, faces = mesh_oracle.extract(keys, tsdf, weight, color, h)
    verts = (verts.astype(f64) - (n - 1) / 2 * h).astype(f32)
    return verts, cols, faces
