"""numpy float64 restatement of mesh cleaning (mesh_clean.py; the casmvs_mesh_clean_* kernels of
csrc/mesh_clean.cu), step by step, bit for bit.

Every double operation is rounded to nearest in the order written below (numpy does not
contract), as the kernels do with __dmul_rn / __dadd_rn.  Piece areas are summed with np.add.at,
which applies its items in index order.  Never imported by the product."""
from __future__ import annotations

import math

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from oracle import simplify_oracle as S
from oracle import texture_oracle as T

MAX_HOLE_LIMIT = 128
HOLE_AREA_FRACTION = 0.1
AREA_CHUNK = 1024
FILLED, NO_TRIANGULATION, AREA_GUARD = 1, 2, 3


def face_area(P, faces):
    n = S.face_normals(P, faces)
    return 0.5 * np.sqrt(S.dot(n, n))


def pieces(P, faces):
    """-> dict like mesh_clean.pieces, as numpy arrays."""
    F = len(faces)
    area = face_area(P, faces)
    comp = T.components(T.neighbours(faces), np.zeros(F, np.int32))
    roots, piece, count = np.unique(comp, return_inverse=True, return_counts=True)
    piece = piece.ravel()
    # rank of each face within its piece, in face order -> its chunk of AREA_CHUNK faces
    order = np.argsort(piece, kind="stable")
    rank = np.empty(F, np.int64)
    rank[order] = np.arange(F) - (np.cumsum(count) - count)[piece[order]]
    n_chunks = (count + AREA_CHUNK - 1) // AREA_CHUNK
    first = np.cumsum(n_chunks) - n_chunks
    chunk = first[piece] + rank // AREA_CHUNK
    partial = np.zeros(int(n_chunks.sum()))
    np.add.at(partial, chunk, area)
    parea = np.zeros(len(roots))
    np.add.at(parea, np.repeat(np.arange(len(roots)), n_chunks), partial)
    return dict(face_area=area, comp=comp, roots=roots.astype(np.int32), count=count, area=parea,
                piece=piece)


def piece_threshold(count, min_faces, min_ratio):
    return max(int(min_faces), math.ceil(min_ratio * int(count.max())))


def boundary_loops(faces, V):
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    ek, _, _, inv, cnt = S.edges(f)
    bnd = cnt[inv] == 1
    A = f.ravel()[bnd]
    B = np.roll(f, -1, 1).ravel()[bnd]
    face = (np.arange(3 * len(f)) // 3)[bnd]
    out_deg = np.bincount(A, minlength=V).astype(np.int32)
    in_deg = np.bincount(B, minlength=V).astype(np.int32)
    nxt = np.full(V, -1, np.int32)
    nface = np.full(V, -1, np.int32)
    ok = (out_deg[A] == 1) & (in_deg[A] == 1)
    nxt[A[ok]], nface[A[ok]] = B[ok], face[ok]
    # components of v -- next[v] over the vertices with next >= 0, named by their least vertex
    on = nxt >= 0
    e = on & on[np.maximum(nxt, 0)]
    src = np.nonzero(e)[0]
    G = coo_matrix((np.ones(len(src)), (src, nxt[src])), shape=(V, V))
    _, lab = connected_components(G, directed=False)
    root = np.full(lab.max() + 1, V, np.int64)
    np.minimum.at(root, lab, np.arange(V))
    comp = np.where(on, root[lab], np.arange(V)).astype(np.int32)
    size = np.bincount(comp[on], minlength=V).astype(np.int32)
    opn = np.zeros(V, np.uint8)
    path = on & ~on[np.maximum(nxt, 0)]
    opn[comp[path]] = 1
    owners = np.nonzero(on & (comp == np.arange(V)) & (opn == 0))[0].astype(np.int32)
    junction = (out_deg != 1) | (in_deg != 1)
    return dict(edge_keys=ek, out_deg=out_deg, in_deg=in_deg, next=nxt, next_face=nface,
                comp=comp, size=size, open=opn, owners=owners, sizes=size[owners],
                not_simple=int(out_deg[junction].sum()))


def loop_vertices(nxt, owner, n):
    vid = [int(owner)]
    for _ in range(n - 1):
        vid.append(int(nxt[vid[-1]]))
    return np.array(vid, np.int64)


def triangulate(P, vid, edge_keys):
    """Minimum-area DP over the loop vid -> (area, triangles (n-2, 3) or None)."""
    n = len(vid)
    p = P.astype(np.float64)[vid]
    cost = np.full((n, n), np.inf)
    split = np.zeros((n, n), np.int64)
    cost[np.arange(n - 1), np.arange(1, n)] = 0.0
    i, j = np.triu_indices(n, 2)
    key = (np.minimum(vid[i], vid[j]) << 32) | np.maximum(vid[i], vid[j])
    pos = np.minimum(np.searchsorted(edge_keys, key), max(len(edge_keys) - 1, 0))
    taken = np.zeros((n, n), bool)
    taken[i, j] = (edge_keys[pos] == key) if len(edge_keys) else False
    taken[0, n - 1] = False
    for d in range(2, n):
        ii = np.arange(n - d)
        jj = ii + d
        kk = ii[:, None] + 1 + np.arange(d - 1)[None, :]
        pi, pj = p[ii][:, None], p[jj][:, None]
        m = S.cross(p[kk] - pi, pj - pi)
        c = (cost[ii[:, None], kk] + cost[kk, jj[:, None]]) + 0.5 * np.sqrt(S.dot(m, m))
        c[(m == 0).all(-1)] = np.inf
        best = np.argmin(c, 1)
        cb = c[np.arange(len(ii)), best]
        good = (cb < np.inf) & ~taken[ii, jj]
        cost[ii[good], jj[good]] = cb[good]
        split[ii[good], jj[good]] = kk[good, best[good]]
    total = cost[0, n - 1]
    if not total < np.inf:
        return total, None
    tris, stack = [], [(0, n - 1)]
    while stack:
        a, b = stack.pop()
        if b - a < 2:
            continue
        k = split[a, b]
        tris.append((vid[b], vid[k], vid[a]))
        stack.append((k, b))
        stack.append((a, k))
    return total, np.array(tris, np.int32)


def fill_holes(P, lp, owners, sizes, piece_area):
    """-> (status (L,) u8, area (L,) f64, tris (sum (n-2), 3) int32 with -1 rows for status 2)."""
    status = np.zeros(len(owners), np.uint8)
    area = np.zeros(len(owners))
    out = []
    for L, (o, n) in enumerate(zip(owners, sizes)):
        total, tris = triangulate(P, loop_vertices(lp["next"], o, int(n)), lp["edge_keys"])
        area[L] = total
        if tris is None:
            status[L] = NO_TRIANGULATION
            out.append(np.full((n - 2, 3), -1, np.int32))
            continue
        status[L] = FILLED if total <= HOLE_AREA_FRACTION * piece_area[lp["next_face"][o]] else AREA_GUARD
        out.append(tris)
    return status, area, (np.concatenate(out) if out else np.zeros((0, 3), np.int32))


def clean_mesh(verts, colours, faces, min_faces=0, min_ratio=0.01, max_hole=0, trace=None):
    """The whole cleaning -> (verts, colours, faces, stats); `trace`, a dict, receives each step's
    state."""
    P = np.asarray(verts, np.float32).reshape(-1, 3)
    C = np.asarray(colours, np.uint8).reshape(-1, 3)
    f0 = np.asarray(faces, np.int64).reshape(-1, 3)
    keep0 = S.clean(P, f0)
    f = f0[keep0].astype(np.int32)
    pc = pieces(P, f)
    thr = piece_threshold(pc["count"], min_faces, min_ratio)
    keep_piece = pc["count"] >= thr
    keep = keep_piece[pc["piece"]]
    f = f[keep]
    stats = dict(faces_in=len(f0), degenerate=int((~keep0).sum()), pieces=len(pc["roots"]),
                 pieces_removed=int((~keep_piece).sum()),
                 faces_removed=int(pc["count"][~keep_piece].sum()), loops=0, loops_not_simple=0,
                 holes_filled=0, holes_too_large=0, holes_no_triangulation=0, holes_area_guard=0,
                 faces_added=0)
    if trace is not None:
        trace.update(cleaned=f0[keep0].astype(np.int32), pieces=pc, kept=f)
    if max_hole >= 3:
        lp = boundary_loops(f, len(P))
        small = lp["sizes"] <= max_hole
        owners, sizes = lp["owners"][small], lp["sizes"][small]
        status, area, tris = fill_holes(P, lp, owners, sizes, pc["area"][pc["piece"][keep]])
        row_loop = np.repeat(np.arange(len(owners)), sizes - 2)
        added = tris[status[row_loop] == FILLED]
        f = np.concatenate([f, added])
        stats.update(loops=len(lp["owners"]), loops_not_simple=lp["not_simple"],
                     holes_filled=int((status == FILLED).sum()), holes_too_large=int((~small).sum()),
                     holes_no_triangulation=int((status == NO_TRIANGULATION).sum()),
                     holes_area_guard=int((status == AREA_GUARD).sum()), faces_added=len(added))
        if trace is not None:
            trace.update(loops=lp, owners=owners, sizes=sizes, status=status, area=area, tris=tris)
    V, Cc, F = S.compact(P, C, f)
    stats.update(vertices=len(V), faces=len(F))
    return V, Cc, F, stats
