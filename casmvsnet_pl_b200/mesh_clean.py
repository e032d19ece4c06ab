"""Clean a triangle mesh on the GPU: drop small disconnected pieces and fill small holes
(csrc/mesh_clean.cu; numpy float64 restatement in oracle/mesh_clean_oracle.py, bit for bit).

    verts, colours, faces, stats = clean_mesh(verts, colours, faces,
                                              min_faces=0, min_ratio=0.01, max_hole=0)

    python -m casmvsnet_pl_b200.mesh_clean --ply in.ply --out out.ply [--min_faces N]
                                           [--min_ratio R] [--max_hole E]

The rule (include/casmvs.h states every operation):
1. cleanup: faces with a repeated index or a zero cross product in double are dropped
   (casmvs_simplify_clean);
2. pieces: a piece is a set of faces joined across manifold edges (texture.neighbours, components
   by casmvs_texture_charts with one label), named by its least face.  Its area is the sum of its
   faces' areas 0.5 |(p1 - p0) x (p2 - p0)| in double, in face order: each chunk of AREA_CHUNK
   consecutive faces of the piece is summed left to right, then the chunk sums left to right.  A piece survives when it
   has at least max(min_faces, ceil(min_ratio x the largest piece's faces)) faces;
3. boundary loops (only when max_hole >= 3): a boundary half-edge is a face's directed edge a -> b
   whose undirected edge has one face.  Where a vertex has one boundary half-edge out and one in,
   next[a] = b.  A simple loop is a cycle of next through such vertices only, owned by its least
   vertex; its positions 0..n-1 start at the owner and follow next.  A loop of n <= max_hole edges
   is a hole; longer ones (the open border of a scene) are counted as too large.  Boundary paths
   that leave a vertex of in- or out-degree other than 1 are counted as not simple, one per
   half-edge out of such a vertex (two for a figure-eight), and never filled;
4. triangulation: the minimum-area triangulation of the loop's vertices (Liepa 2003, area term
   only) by O(n^3) dynamic programming in double, least split index on equal cost, never using a
   triangle with a zero cross product or a diagonal that is already a mesh edge.  A loop without
   an admissible triangulation is skipped and counted.  Each fill triangle lists its loop
   positions in decreasing order, so every boundary half-edge meets its reversed twin;
5. area guard: a hole is filled only when its triangulation's area is at most HOLE_AREA_FRACTION
   of the area of the piece holding its owner's outgoing boundary half-edge, so a surviving disc is
   not capped by a second disc, nor an isolated triangle by its twin;
6. output: surviving faces keep their input order; the fill faces follow in owner order, each
   loop's in the DP's pre-order (the triangle on (0, n-1) first, then the part left of its split,
   then the part right of it).  Vertices no face references are removed; the rest keep their
   order and colours.  No vertex is added.

Properties: a fill edge is never non-manifold (loops share no vertex, and a diagonal is never an
existing edge); a closed piece is untouched (it has no boundary); a planar convex hole is filled
with exactly its polygon area (every triangulation of a planar convex polygon has that area, up to
rounding)."""
from __future__ import annotations

import argparse
import ctypes
import math

import numpy as np
import torch

from . import _lib, io, mesh, simplify, texture

MAX_HOLE_LIMIT = 128
HOLE_AREA_FRACTION = 0.1
AREA_CHUNK = 1024
# device bytes: per input face the cleaned faces, the neighbour table with its int64 keys and
# sorts, the components, areas and piece sort, and the edge topology of the surviving faces; per
# vertex the boundary degrees, next, the loop components and the compaction.  bench_mesh_clean.py
# measured a peak of 309 to 315 bytes per input face (about two faces per vertex) on an H100
BYTES_PER_FACE = 300
BYTES_PER_VERTEX = 64
STATUS_FILLED, STATUS_NO_TRIANGULATION, STATUS_AREA_GUARD = 1, 2, 3


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def cleanup(verts, faces):
    """Step 1 -> (faces without degenerate ones (F', 3) int32, dropped count)."""
    keep = torch.empty(len(faces), dtype=torch.uint8, device=verts.device)
    _lib.check(_lib.load().casmvs_simplify_clean(_ptr(verts), _ptr(faces), len(faces), _ptr(keep),
                                                 _stream()), "simplify_clean")
    f = faces[keep.bool()].contiguous()
    return f, len(faces) - len(f)


def pieces(verts, faces, mark=None):
    """Step 2's pieces -> dict: face_area (F,) f64, comp (F,) int32 (least face of the piece),
    roots (P,) int32 ascending, count (P,) int64, area (P,) f64, piece (F,) int64 (row in roots).
    `mark`, when given, is called with "pieces" once the components are known."""
    lib = _lib.load()
    F, dev = len(faces), verts.device
    comp, _ = texture.components(texture.neighbours(faces),
                                 torch.zeros(F, dtype=torch.int32, device=dev))
    if mark:
        mark("pieces")
    area = torch.empty(F, dtype=torch.float64, device=dev)
    _lib.check(lib.casmvs_mesh_clean_face_area(_ptr(verts), _ptr(faces), F, _ptr(area), _stream()),
               "mesh_clean_face_area")
    sc, order = torch.sort(comp, stable=True)
    roots, count = torch.unique_consecutive(sc, return_counts=True)
    # chunks of up to AREA_CHUNK consecutive faces of a piece, bounds in `order` positions
    n_chunks = (count + AREA_CHUNK - 1) // AREA_CHUNK
    piece_chunks = torch.zeros(len(roots) + 1, dtype=torch.int64, device=dev)
    piece_chunks[1:] = torch.cumsum(n_chunks, 0)
    chunk_piece = torch.repeat_interleave(torch.arange(len(roots), device=dev), n_chunks)
    bounds = torch.full((len(chunk_piece) + 1,), F, dtype=torch.int64, device=dev)
    bounds[:-1] = (torch.cumsum(count, 0) - count)[chunk_piece] + AREA_CHUNK * (
        torch.arange(len(chunk_piece), device=dev) - piece_chunks[chunk_piece])
    partial = torch.empty(len(chunk_piece), dtype=torch.float64, device=dev)
    parea = torch.empty(len(roots), dtype=torch.float64, device=dev)
    _lib.check(lib.casmvs_mesh_clean_sums(_ptr(area), _ptr(order), _ptr(bounds), len(partial),
                                          _ptr(partial), _stream()), "mesh_clean_sums")
    _lib.check(lib.casmvs_mesh_clean_sums(_ptr(partial), None, _ptr(piece_chunks), len(roots),
                                          _ptr(parea), _stream()), "mesh_clean_sums")
    return dict(face_area=area, comp=comp, roots=roots, count=count, area=parea,
                piece=torch.searchsorted(roots, comp))


def piece_threshold(count, min_faces, min_ratio):
    """The least face count of a surviving piece: max(min_faces, ceil(min_ratio x largest))."""
    return max(int(min_faces), math.ceil(min_ratio * int(count.max())))


def boundary_loops(faces, V):
    """Step 3's boundary -> dict: edge_keys (E,) int64 of `faces`, out_deg / in_deg (V,) int32,
    next / next_face (V,) int32 (-1 off simple boundary vertices), comp (V,) int32, size (V,)
    int32, open (V,) u8, owners (L,) int32 ascending and sizes (L,) int32 of the simple loops, and
    not_simple, the boundary half-edges out of vertices of in- or out-degree other than 1."""
    lib = _lib.load()
    dev = faces.device
    ek, inv, cnt, _, _ = simplify._topology(faces, V)
    d = {k: torch.empty(V, dtype=torch.int32, device=dev)
         for k in ("out_deg", "in_deg", "next", "next_face", "size")}
    _lib.check(lib.casmvs_mesh_clean_boundary(_ptr(faces), len(faces), _ptr(inv), _ptr(cnt), V,
                                              _ptr(d["out_deg"]), _ptr(d["in_deg"]), _ptr(d["next"]),
                                              _ptr(d["next_face"]), _stream()), "mesh_clean_boundary")
    nbr = torch.full((V, 3), -1, dtype=torch.int32, device=dev)
    nbr[:, 0] = d["next"]
    label = torch.where(d["next"] >= 0, 0, -1).int()
    comp, _ = texture.components(nbr, label)
    opn = torch.empty(V, dtype=torch.uint8, device=dev)
    _lib.check(lib.casmvs_mesh_clean_loop_sizes(_ptr(d["next"]), _ptr(comp), V, _ptr(d["size"]),
                                                _ptr(opn), _stream()), "mesh_clean_loop_sizes")
    ar = torch.arange(V, dtype=torch.int32, device=dev)
    owners = torch.nonzero((d["next"] >= 0) & (comp == ar) & (opn == 0)).squeeze(1).int()
    junction = (d["out_deg"] != 1) | (d["in_deg"] != 1)
    return dict(d, edge_keys=ek, comp=comp, open=opn, owners=owners, sizes=d["size"][owners],
                not_simple=int(d["out_deg"][junction].sum()))


def fill_holes(verts, lp, owners, sizes, piece_area):
    """Steps 4-5 for the loops `owners` / `sizes` (each 3..MAX_HOLE_LIMIT) of boundary_loops' `lp`,
    piece_area (F,) f64 per face -> (status (L,) u8, area (L,) f64, tris (sum (n - 2), 3) int32,
    the loop of each triangle row (int64))."""
    dev = verts.device
    n_tri = (sizes - 2).long()
    tri_off = torch.cumsum(n_tri, 0) - n_tri
    tris = torch.empty(int(n_tri.sum()), 3, dtype=torch.int32, device=dev)
    status = torch.empty(len(owners), dtype=torch.uint8, device=dev)
    area = torch.empty(len(owners), dtype=torch.float64, device=dev)
    max_size = int(sizes.max()) if len(sizes) else 0
    _lib.check(_lib.load().casmvs_mesh_clean_fill(
        _ptr(verts), _ptr(lp["next"]), _ptr(lp["next_face"]), _ptr(owners), _ptr(sizes), len(owners),
        max_size, _ptr(tri_off), _ptr(lp["edge_keys"]), len(lp["edge_keys"]), _ptr(piece_area),
        _ptr(status), _ptr(area), _ptr(tris), _stream()), "mesh_clean_fill")
    row_loop = torch.repeat_interleave(torch.arange(len(owners), device=dev), n_tri)
    return status, area, tris, row_loop


def _check_inputs(verts, colours, faces, min_faces, min_ratio, max_hole):
    if isinstance(min_faces, bool) or not isinstance(min_faces, (int, np.integer)) or min_faces < 0:
        raise ValueError(f"min_faces must be an integer >= 0, got {min_faces!r}")
    if isinstance(min_ratio, bool) or not isinstance(min_ratio, (int, float, np.floating, np.integer)) \
            or not 0 <= min_ratio <= 1:
        raise ValueError(f"min_ratio must be a number in [0, 1], got {min_ratio!r}")
    if isinstance(max_hole, bool) or not isinstance(max_hole, (int, np.integer)) \
            or not (max_hole == 0 or 3 <= max_hole <= MAX_HOLE_LIMIT):
        raise ValueError(f"max_hole must be 0 (no filling) or an integer in 3..{MAX_HOLE_LIMIT}, "
                         f"got {max_hole!r}")
    for name, t, dtypes in (("verts", verts, (torch.float32,)), ("colours", colours, (torch.uint8,)),
                            ("faces", faces, (torch.int32, torch.int64))):
        if not (torch.is_tensor(t) and t.is_cuda and t.dtype in dtypes and t.dim() == 2
                and t.shape[1] == 3):
            raise ValueError(f"{name} must be a CUDA tensor of shape (N, 3) and dtype "
                             f"{' or '.join(map(str, dtypes))}")
    if len(colours) != len(verts):
        raise ValueError(f"colours has {len(colours)} rows but verts has {len(verts)}")
    if not (colours.device == faces.device == verts.device):
        raise ValueError("verts, colours and faces must be on one device")
    if len(faces) == 0:
        raise ValueError("the mesh has no faces")
    if 3 * max(len(verts), len(faces)) >= 2 ** 31:
        raise ValueError(f"a mesh of {len(verts)} vertices and {len(faces)} faces is too large "
                         "(3 x either must stay below 2^31)")
    if not bool(torch.isfinite(verts).all()):
        raise ValueError("verts holds a non-finite coordinate")
    if not bool(((faces >= 0) & (faces < len(verts))).all()):
        raise ValueError(f"faces holds an index outside 0..{len(verts) - 1}")


def clean_mesh(verts, colours, faces, min_faces=0, min_ratio=0.01, max_hole=0, max_bytes=None):
    """Drop the pieces of fewer than max(min_faces, ceil(min_ratio x the largest piece's faces))
    faces and, when max_hole >= 3, fill the holes of at most max_hole edges (verts (N,3) float32,
    colours (N,3) uint8, faces (M,3) int32 or int64, CUDA tensors) -> (verts, colours, faces int32,
    stats: faces_in, degenerate, pieces, pieces_removed, faces_removed, loops, loops_not_simple,
    holes_filled, holes_too_large, holes_no_triangulation, holes_area_guard, faces_added,
    vertices, faces).  Raises ValueError on bad input or when nothing would be left, CasMVSError
    when the work would not fit in mesh.device_budget."""
    _check_inputs(verts, colours, faces, min_faces, min_ratio, max_hole)
    dev = verts.device
    need = len(faces) * BYTES_PER_FACE + len(verts) * BYTES_PER_VERTEX
    with torch.cuda.device(dev):
        budget = mesh.device_budget(dev, max_bytes)
        if need > budget:
            raise _lib.CasMVSError(
                f"cleaning {len(faces)} faces and {len(verts)} vertices needs {need} bytes of "
                f"device memory but {max(budget, 0)} bytes are available")
        P, C = verts.contiguous(), colours.contiguous()
        f, degenerate = cleanup(P, faces.int().contiguous())
        if len(f) == 0:
            raise ValueError("cleaning would leave no faces: every face is degenerate")
        pc = pieces(P, f)
        thr = piece_threshold(pc["count"], min_faces, min_ratio)
        keep_piece = pc["count"] >= thr
        if not bool(keep_piece.any()):
            raise ValueError(f"cleaning would leave no faces: min_faces {min_faces} exceeds the "
                             f"largest piece's {int(pc['count'].max())} faces")
        keep = keep_piece[pc["piece"]]
        f = f[keep].contiguous()
        stats = dict(faces_in=len(faces), degenerate=degenerate, pieces=len(pc["roots"]),
                     pieces_removed=int((~keep_piece).sum()),
                     faces_removed=int(pc["count"][~keep_piece].sum()), loops=0,
                     loops_not_simple=0, holes_filled=0, holes_too_large=0,
                     holes_no_triangulation=0, holes_area_guard=0, faces_added=0)
        if max_hole >= 3:
            lp = boundary_loops(f, len(P))
            small = lp["sizes"] <= max_hole
            owners, sizes = lp["owners"][small], lp["sizes"][small]
            status, _, tris, row_loop = fill_holes(P, lp, owners, sizes,
                                                   pc["area"][pc["piece"][keep]])
            added = tris[status[row_loop] == STATUS_FILLED]
            f = torch.cat([f, added]).contiguous()
            stats.update(loops=len(lp["owners"]), loops_not_simple=lp["not_simple"],
                         holes_filled=int((status == STATUS_FILLED).sum()),
                         holes_too_large=int((~small).sum()),
                         holes_no_triangulation=int((status == STATUS_NO_TRIANGULATION).sum()),
                         holes_area_guard=int((status == STATUS_AREA_GUARD).sum()),
                         faces_added=len(added))
        V, Cc, F = simplify._compact(P, C, f)
    stats.update(vertices=len(V), faces=len(F))
    return V, Cc, F, stats


def summary(st):
    """One line of the stats."""
    return (f"{st['faces_in']} -> {st['faces']} faces: {st['degenerate']} degenerate, "
            f"{st['pieces_removed']} of {st['pieces']} pieces removed ({st['faces_removed']} faces), "
            f"{st['holes_filled']} of {st['loops']} loops filled ({st['faces_added']} faces; "
            f"{st['holes_too_large']} too large, {st['holes_no_triangulation']} without a "
            f"triangulation, {st['holes_area_guard']} over the area guard, "
            f"{st['loops_not_simple']} not simple)")


def _parser():
    ap = argparse.ArgumentParser(description="Clean a triangle-mesh PLY on the GPU: drop small "
                                             "disconnected pieces and fill small holes.")
    ap.add_argument("--ply", required=True, help="the mesh to clean (binary PLY, as mesh.py and "
                                                 "poisson.py write)")
    ap.add_argument("--out", required=True, help="the cleaned mesh PLY to write")
    ap.add_argument("--min_faces", type=int, default=0,
                    help="drop pieces of fewer faces than this (>= 0, default 0)")
    ap.add_argument("--min_ratio", type=float, default=0.01,
                    help="drop pieces of fewer faces than this fraction of the largest piece's, "
                         "rounded up (in [0, 1], default 0.01)")
    ap.add_argument("--max_hole", type=int, default=0,
                    help=f"fill holes of at most this many boundary edges (0: none, or "
                         f"3..{MAX_HOLE_LIMIT}; default 0)")
    return ap


def parse_args(argv=None):
    ap = _parser()
    a = ap.parse_args(argv)
    if a.min_faces < 0:
        ap.error("--min_faces must be >= 0")
    if not (math.isfinite(a.min_ratio) and 0 <= a.min_ratio <= 1):
        ap.error("--min_ratio must be in [0, 1]")
    if not (a.max_hole == 0 or 3 <= a.max_hole <= MAX_HOLE_LIMIT):
        ap.error(f"--max_hole must be 0 or in 3..{MAX_HOLE_LIMIT}")
    return a


def main(argv=None):
    a = parse_args(argv)
    v, c, f = io.read_mesh_ply(a.ply)
    dev = torch.device("cuda", torch.cuda.current_device())
    V, C, F, st = clean_mesh(torch.from_numpy(np.ascontiguousarray(v)).to(dev),
                             torch.from_numpy(np.ascontiguousarray(c)).to(dev),
                             torch.from_numpy(np.ascontiguousarray(f)).to(dev),
                             min_faces=a.min_faces, min_ratio=a.min_ratio, max_hole=a.max_hole)
    mesh.write_mesh_ply(a.out, V, C, F)
    print(f"{a.ply}: {summary(st)}; wrote {a.out}")


if __name__ == "__main__":
    main()
