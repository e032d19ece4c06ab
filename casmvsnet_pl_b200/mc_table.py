"""The marching-cubes case table of csrc/mesh.cu, generated from one rule instead of typed in.

Cube corners are numbered c = x + 2y + 4z (x, y, z in {0, 1}); a corner is inside when its TSDF
value is < 0 and case = sum of 1 << c over the inside corners.  Edge e = 4 * axis + k runs along
`axis` from its lower corner, whose other two coordinates are the bits of k (low bit: the lower
of the two other axes), to that corner + (1 << axis).

The rule, per case:
  * On each of the six cube faces, the face's crossing edges (one inside and one outside corner)
    are joined by segments: two crossings by one segment; four crossings (an ambiguous face,
    diagonal corners equal) by two segments that each cut off one INSIDE corner.  The rule reads
    the face's four signs only, so the two cells sharing a face join its crossings the same way
    and the mesh is watertight.
  * Each segment is directed so that, seen from outside the cube through its face, the inside
    corners lie to its right; then the loop it belongs to runs counter-clockwise around the
    normal that points from inside to outside (towards free space).
  * Every crossing edge lies on two faces, so it ends one segment and starts another: the segments
    chain into closed loops, taken in order of their smallest edge.  Each loop is fan-triangulated
    from the first of its vertices (in loop order from the smallest edge) from which no diagonal
    joins two edges of one cube face; such a diagonal could be drawn by both cells of that face.

    python -m casmvsnet_pl_b200.mc_table        # rewrites csrc/mc_table.h
"""
from __future__ import annotations

import os

import numpy as np

HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "mc_table.h")


def corner_pos(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], dtype=np.float64)


def edge_corners(e):
    """-> (lower corner, upper corner) of edge e."""
    axis, k = divmod(e, 4)
    o0, o1 = [a for a in range(3) if a != axis]
    c0 = ((k & 1) << o0) | ((k >> 1) << o1)
    return c0, c0 | (1 << axis)


EDGES = [edge_corners(e) for e in range(12)]
_EDGE_OF = {frozenset(EDGES[e]): e for e in range(12)}


def faces():
    """[(corners in cyclic order, outward normal)] of the six cube faces."""
    out = []
    for axis in range(3):
        o0, o1 = [a for a in range(3) if a != axis]
        for side in (0, 1):
            def corner(u, v):
                return (side << axis) | (u << o0) | (v << o1)
            n = np.zeros(3)
            n[axis] = 1.0 if side else -1.0
            out.append(([corner(0, 0), corner(1, 0), corner(1, 1), corner(0, 1)], n))
    return out


FACES = faces()
_FACE_SETS = [frozenset(cyc) for cyc, _ in FACES]


def _mid(e):
    a, b = EDGES[e]
    return 0.5 * (corner_pos(a) + corner_pos(b))


def face_segments(case):
    """Directed segments (edge_from, edge_to) of every face for `case`."""
    segs = []
    for cyc, n in FACES:
        ins = [(case >> c) & 1 for c in cyc]
        cross = [i for i in range(4) if ins[i] != ins[(i + 1) % 4]]   # side i: cyc[i] - cyc[i+1]
        side_edge = [_EDGE_OF[frozenset((cyc[i], cyc[(i + 1) % 4]))] for i in range(4)]
        pairs = []
        if len(cross) == 2:
            a, b = side_edge[cross[0]], side_edge[cross[1]]
            pin = np.mean([corner_pos(c) for c, s in zip(cyc, ins) if s], axis=0)
            pout = np.mean([corner_pos(c) for c, s in zip(cyc, ins) if not s], axis=0)
            pairs.append((a, b, pout - pin))
        elif len(cross) == 4:
            for i in range(4):
                if ins[i]:                          # cut off inside corner cyc[i]
                    a, b = side_edge[(i - 1) % 4], side_edge[i]
                    pairs.append((a, b, 0.5 * (_mid(a) + _mid(b)) - corner_pos(cyc[i])))
        for a, b, g in pairs:
            d = _mid(b) - _mid(a)
            if np.dot(np.cross(g, d), n) > 0:
                a, b = b, a
            segs.append((a, b))
    return segs


def _share_face(e0, e1):
    s = frozenset(EDGES[e0]) | frozenset(EDGES[e1])
    return any(s <= f for f in _FACE_SETS)


def case_loops(case):
    """Closed loops of edge indices, each in its oriented order starting at its smallest edge."""
    nxt = {}
    for a, b in face_segments(case):
        if a in nxt:
            raise AssertionError(f"case {case}: edge {a} starts two segments")
        nxt[a] = b
    if sorted(nxt) != sorted(nxt.values()):
        raise AssertionError(f"case {case}: segments do not chain")
    loops, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        if e != start:
            raise AssertionError(f"case {case}: open loop {loop}")
        loops.append(loop)
    return loops


def _fan(loop):
    n = len(loop)
    for r in range(n):
        lp = loop[r:] + loop[:r]
        if all(not _share_face(lp[0], lp[k]) for k in range(2, n - 1)):
            return [(lp[0], lp[k], lp[k + 1]) for k in range(1, n - 1)]
    raise AssertionError(f"loop {loop}: every fan apex has a diagonal on a cube face")


def case_triangles(case):
    return [t for loop in case_loops(case) for t in _fan(loop)]


def table():
    """-> (tris (256, max_tris, 3) int8 padded with -1, count (256,) int, edge_mask (256,) int)."""
    tris = [case_triangles(c) for c in range(256)]
    width = max(len(t) for t in tris)
    out = np.full((256, width, 3), -1, dtype=np.int8)
    for c, ts in enumerate(tris):
        if ts:
            out[c, :len(ts)] = ts
    count = np.array([len(t) for t in tris], dtype=np.int64)
    mask = np.array([sum(1 << e for e in {e for t in ts for e in t}) for ts in tris], dtype=np.int64)
    return out, count, mask


def header_text():
    tris, count, mask = table()
    width = tris.shape[1]
    lines = ["// Marching-cubes case table of mesh.cu.  Generated by casmvsnet_pl_b200/mc_table.py",
             "// (the rule is documented there); do not edit: a CPU test keeps it in sync.",
             "#pragma once", "",
             f"#define CASMVS_MC_MAX_TRIS {width}", "",
             "// triangles per case",
             "__device__ const unsigned char kMcTriCount[256] = {"]
    for r in range(0, 256, 16):
        lines.append("    " + ", ".join(str(int(v)) for v in count[r:r + 16]) + ",")
    lines += ["};", "", "// bit e set: edge e is a crossing edge of the case",
              "__device__ const unsigned short kMcEdgeMask[256] = {"]
    for r in range(0, 256, 8):
        lines.append("    " + ", ".join(f"0x{int(v):03x}" for v in mask[r:r + 8]) + ",")
    lines += ["};", "",
              "// edges of each triangle, counter-clockwise seen from outside (tsdf >= 0); -1 pads",
              f"__device__ const signed char kMcTris[256][{3 * width}] = {{"]
    for c in range(256):
        lines.append("    {" + ", ".join(str(int(v)) for v in tris[c].reshape(-1)) + "},")
    lines += ["};", ""]
    return "\n".join(lines)


def main():
    with open(HEADER, "w") as f:
        f.write(header_text())
    print(f"wrote {HEADER}")


if __name__ == "__main__":
    main()
