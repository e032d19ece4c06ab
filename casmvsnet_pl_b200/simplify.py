"""Simplify a triangle mesh on the GPU: quadric edge-collapse decimation (Garland & Heckbert
1997) to a face budget, in parallel rounds of independent collapses (csrc/simplify.cu; numpy
float64 restatement in oracle/simplify_oracle.py, bit for bit).

    verts, colours, faces, stats = simplify_mesh(verts, colours, faces, target_faces=100_000)

    python -m casmvsnet_pl_b200.simplify --ply in.ply --out out.ply (--faces N | --ratio R)
                                         [--max_error E]

The rule (include/casmvs.h states every operation):
- once: faces with a repeated index or zero area are dropped; vertices on an edge of > 2 faces,
  with > MAX_FAN faces or whose faces are not one fan are frozen; each vertex takes the sum of its
  faces' area-weighted plane quadrics and of BOUNDARY_WEIGHT |e|^2 times the quadric of the plane
  through each boundary edge perpendicular to its face;
- per round: the unique edges and the vertex -> face CSR are rebuilt; every edge gets the
  optimal position of Q_a + Q_b (or the best of a, b, midpoint when A is singular), its cost,
  validity (link condition, no pinched boundary, >= 3 neighbours kept, fan <= MAX_FAN, no face
  folding past cos 0.2, cost <= max_error) and key (cost bits << 32 | edge index); the candidates
  are the valid edges with key <= the ceil(E_valid / CANDIDATE_DIVISOR)-th smallest; an edge is
  collapsed when its key is the least over the 1-rings of both endpoints; the selection is cut to
  the key-ordered prefix that reaches the target, then the lower index survives at the new
  position.
Rounds repeat until F <= target, no edge is valid, or (with max_error) every valid edge costs
more.  The result has target or target - 1 faces unless it stops early; surviving vertices and
faces keep their input order."""
from __future__ import annotations

import argparse
import ctypes
import math

import numpy as np
import torch

from . import _lib, io, mesh

MAX_FAN = 32
BOUNDARY_WEIGHT = 1000.0
CANDIDATE_DIVISOR = 4
# device bytes: per input face the faces, corner keys and the sorts of a round (~260), the
# edges' keys, positions, costs and flags at up to 1.5 edges per face (~60) and the face quadrics
# of the set-up (80); per vertex the position, colour, quadric, flags and the selection minima
BYTES_PER_FACE = 400
BYTES_PER_VERTEX = 160
_KEY_NONE = torch.iinfo(torch.int64).max


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _topology(faces, V):
    """-> (edge keys (E,) int64 sorted, corner -> edge (3F,) int32, faces per edge (E,) int32,
    CSR offsets (V+1,) int32, corners in vertex then face order (3F,) int32)."""
    f = faces.long()
    g = f.roll(-1, 1)
    key = (torch.minimum(f, g) << 32) | torch.maximum(f, g)
    ek, inv, cnt = torch.unique(key.reshape(-1), sorted=True, return_inverse=True,
                                return_counts=True)
    flat, corners = torch.sort(f.reshape(-1), stable=True)
    off = torch.searchsorted(flat, torch.arange(V + 1, device=f.device)).int()
    return ek, inv.int(), cnt.int(), off, corners.int()


def _prepare(verts, colours, faces):
    """Input cleanup, frozen flags and vertex quadrics -> (P, C, faces, frozen, Q, dropped)."""
    lib = _lib.load()
    P, C = verts.clone(), colours.clone()
    V = len(P)
    keep = torch.empty(len(faces), dtype=torch.uint8, device=P.device)
    _lib.check(lib.casmvs_simplify_clean(_ptr(P), _ptr(faces), len(faces), _ptr(keep), _stream()),
               "simplify_clean")
    f = faces[keep.bool()].contiguous()
    dropped = len(faces) - len(f)
    ek, inv, cnt, off, corners = _topology(f, V)
    frozen = torch.empty(V, dtype=torch.uint8, device=P.device)
    _lib.check(lib.casmvs_simplify_frozen(_ptr(f), V, _ptr(off), _ptr(corners), _ptr(inv),
                                          _ptr(cnt), _ptr(frozen), _stream()), "simplify_frozen")
    fq = torch.empty(len(f), 10, dtype=torch.float64, device=P.device)
    _lib.check(lib.casmvs_simplify_face_quadrics(_ptr(P), _ptr(f), len(f), _ptr(fq), _stream()),
               "simplify_face_quadrics")
    Q = torch.empty(V, 10, dtype=torch.float64, device=P.device)
    _lib.check(lib.casmvs_simplify_vertex_quadrics(
        _ptr(P), _ptr(f), V, _ptr(off), _ptr(corners), _ptr(inv), _ptr(ek), _ptr(cnt), _ptr(fq),
        _ptr(Q), _stream()), "simplify_vertex_quadrics")
    return P, C, f, frozen, Q, dropped


def _round_state(P, Q, faces, frozen, max_error=None):
    """Edges, CSR, positions, costs, validity and keys of the current mesh (steps 1-3 of a round)."""
    return _edge_costs(P, Q, faces, frozen, max_error, _topology(faces, len(P)))


def _edge_costs(P, Q, faces, frozen, max_error, topology):
    lib = _lib.load()
    dev, V = P.device, len(P)
    ek, inv, cnt, off, corners = topology
    E = len(ek)
    st = dict(ek=ek, cnt=cnt, off=off, corners=corners,
              deg=torch.empty(V, dtype=torch.int32, device=dev),
              bnd=torch.empty(V, dtype=torch.uint8, device=dev),
              v=torch.empty(E, 3, dtype=torch.float32, device=dev),
              cost=torch.empty(E, dtype=torch.float32, device=dev),
              valid0=torch.empty(E, dtype=torch.uint8, device=dev),
              key=torch.empty(E, dtype=torch.int64, device=dev))
    _lib.check(lib.casmvs_simplify_edge_costs(
        _ptr(P), _ptr(Q), _ptr(faces), V, _ptr(off), _ptr(corners), _ptr(ek), _ptr(cnt), E,
        _ptr(frozen), int(max_error is not None), float(max_error or 0.0), _ptr(st["deg"]),
        _ptr(st["bnd"]), _ptr(st["v"]), _ptr(st["cost"]), _ptr(st["valid0"]), _ptr(st["key"]),
        _stream()), "simplify_edge_costs")
    return st


def _select(st, faces, V):
    """-> (selected edges (E,) bool, threshold key), or (None, None) when no edge is valid."""
    key = st["key"]
    n_valid = int((key != _KEY_NONE).sum())
    if n_valid == 0:
        return None, None
    k = (n_valid + CANDIDATE_DIVISOR - 1) // CANDIDATE_DIVISOR
    thr = int(torch.sort(key).values[k - 1])
    dev = key.device
    m1 = torch.empty(V, dtype=torch.int64, device=dev)
    m2 = torch.empty(V, dtype=torch.int64, device=dev)
    sel = torch.empty(len(key), dtype=torch.uint8, device=dev)
    _lib.check(_lib.load().casmvs_simplify_select(
        _ptr(st["ek"]), _ptr(key), len(key), thr, _ptr(faces), V, _ptr(st["off"]),
        _ptr(st["corners"]), _ptr(m1), _ptr(m2), _ptr(sel), _stream()), "simplify_select")
    return sel.bool(), thr


def _budget(st, sel, F, target):
    """Selected edges in key order, cut to the shortest prefix removing >= F - target faces."""
    idx = torch.nonzero(sel).squeeze(1)
    idx = idx[torch.sort(st["key"][idx]).indices]
    removed = torch.cumsum(st["cnt"][idx].long(), 0)
    need = torch.tensor([F - target], dtype=torch.int64, device=idx.device)
    n = min(len(idx), int(torch.searchsorted(removed, need)) + 1)
    return idx[:n].contiguous()


def _collapse(P, C, Q, faces, st, idx):
    """Apply the collapses `idx` to P, C, Q in place -> the compacted faces."""
    lib = _lib.load()
    remap = torch.arange(len(P), dtype=torch.int32, device=P.device)
    _lib.check(lib.casmvs_simplify_collapse(_ptr(st["ek"]), _ptr(idx), len(idx), _ptr(st["v"]),
                                            _ptr(P), _ptr(C), _ptr(Q), _ptr(remap), _stream()),
               "simplify_collapse")
    f = faces.clone()
    keep = torch.empty(len(f), dtype=torch.uint8, device=P.device)
    _lib.check(lib.casmvs_simplify_remap_faces(_ptr(f), len(f), _ptr(remap), _ptr(keep), _stream()),
               "simplify_remap_faces")
    return f[keep.bool()].contiguous()


def _round(P, C, Q, faces, frozen, target, max_error=None):
    """One round on the current mesh (P, C, Q updated in place) -> (faces, info dict: state,
    sel, thr, idx); faces is None when no edge is valid."""
    st = _round_state(P, Q, faces, frozen, max_error)
    sel, thr = _select(st, faces, len(P))
    if sel is None:
        return None, dict(st, sel=None, thr=None, idx=None)
    idx = _budget(st, sel, len(faces), target)
    info = dict(st, sel=sel, thr=thr, idx=idx, max_cost=float(st["cost"][idx].max()))
    return _collapse(P, C, Q, faces, st, idx), info


def _compact(P, C, faces):
    lib = _lib.load()
    V = len(P)
    used = torch.empty(V, dtype=torch.int32, device=P.device)
    _lib.check(lib.casmvs_simplify_mark_used(_ptr(faces), len(faces), V, _ptr(used), _stream()),
               "simplify_mark_used")
    new = (torch.cumsum(used, 0, dtype=torch.int32) - 1).int()
    f = faces.clone()
    keep = torch.empty(len(f), dtype=torch.uint8, device=P.device)
    _lib.check(lib.casmvs_simplify_remap_faces(_ptr(f), len(f), _ptr(new), _ptr(keep), _stream()),
               "simplify_remap_faces")
    u = used.bool()
    return P[u].contiguous(), C[u].contiguous(), f


def _check_inputs(verts, colours, faces, target_faces, max_error):
    if isinstance(target_faces, bool) or not isinstance(target_faces, (int, np.integer)) \
            or target_faces < 1:
        raise ValueError(f"target_faces must be an integer >= 1, got {target_faces!r}")
    if max_error is not None and not (math.isfinite(max_error) and max_error >= 0):
        raise ValueError(f"max_error must be a finite number >= 0, got {max_error!r}")
    for name, t, dtypes in (("verts", verts, (torch.float32,)), ("colours", colours, (torch.uint8,)),
                            ("faces", faces, (torch.int32, torch.int64))):
        if not (torch.is_tensor(t) and t.is_cuda and t.dtype in dtypes and t.dim() == 2
                and t.shape[1] == 3):
            raise ValueError(f"{name} must be a CUDA tensor of shape (N, 3) and dtype "
                             f"{' or '.join(map(str, dtypes))}")
    if len(colours) != len(verts):
        raise ValueError(f"colours has {len(colours)} rows but verts has {len(verts)}")
    if 3 * max(len(verts), len(faces)) >= 2 ** 31:
        raise ValueError(f"a mesh of {len(verts)} vertices and {len(faces)} faces is too large "
                         "(3 x either must stay below 2^31)")
    if len(verts) and not bool(torch.isfinite(verts).all()):
        raise ValueError("verts holds a non-finite coordinate")
    if len(faces) and not bool(((faces >= 0) & (faces < len(verts))).all()):
        raise ValueError(f"faces holds an index outside 0..{len(verts) - 1}")


def simplify_mesh(verts, colours, faces, target_faces, max_error=None, max_bytes=None, log=print):
    """Decimate a mesh (verts (N,3) float32, colours (N,3) uint8, faces (M,3) int32 or int64, CUDA
    tensors, as mesh.extract_bricks returns them) to at most `target_faces` faces (target or
    target - 1 unless it stops early), never collapsing an edge that costs more than `max_error`.
    -> (verts, colours, faces int32, stats: faces_in, vertices_in, faces, vertices, rounds,
    collapses, max_cost, frozen_vertices, dropped_faces, stop = target | no_candidate |
    max_error).  Raises CasMVSError when the work would not fit in mesh.device_budget."""
    _check_inputs(verts, colours, faces, target_faces, max_error)
    dev = verts.device
    need = len(faces) * BYTES_PER_FACE + len(verts) * BYTES_PER_VERTEX
    with torch.cuda.device(dev):
        budget = mesh.device_budget(dev, max_bytes)
        if need > budget:
            raise _lib.CasMVSError(
                f"simplifying {len(faces)} faces and {len(verts)} vertices needs {need} bytes of "
                f"device memory but {max(budget, 0)} bytes are available")
        P, C, f, frozen, Q, dropped = _prepare(verts.contiguous(), colours.contiguous(),
                                               faces.int().contiguous())
        rounds = collapses = 0
        max_cost, stop = 0.0, "target"
        while len(f) > target_faces:
            nf, info = _round(P, C, Q, f, frozen, target_faces, max_error)
            if nf is None:
                stop = ("max_error" if max_error is not None and bool(info["valid0"].any())
                        else "no_candidate")
                break
            f = nf
            rounds += 1
            collapses += len(info["idx"])
            max_cost = max(max_cost, info["max_cost"])
        V, Cc, F = _compact(P, C, f)
    stats = dict(faces_in=len(faces), vertices_in=len(verts), faces=len(F), vertices=len(V),
                 rounds=rounds, collapses=collapses, max_cost=max_cost,
                 frozen_vertices=int(frozen.sum()), dropped_faces=dropped, stop=stop)
    if len(F) > target_faces:
        log(f"simplify: stopped at {len(F)} faces, above the target of {target_faces} "
            f"({'every valid edge costs more than max_error' if stop == 'max_error' else 'no edge can be collapsed'})")
    return V, Cc, F, stats


def _parser():
    ap = argparse.ArgumentParser(description="Simplify a triangle-mesh PLY on the GPU by quadric "
                                             "edge-collapse decimation.")
    ap.add_argument("--ply", required=True, help="the mesh to simplify (binary PLY, as mesh.py "
                                                 "and poisson.py write)")
    ap.add_argument("--out", required=True, help="the simplified mesh PLY to write")
    g = ap.add_mutually_exclusive_group(required=True)
    g.add_argument("--faces", type=int, help="the target number of faces (>= 1)")
    g.add_argument("--ratio", type=float, help="the target as a fraction of the input faces, "
                                               "in (0, 1]: max(1, round(R F))")
    ap.add_argument("--max_error", type=float, default=None,
                    help="never collapse an edge whose quadric cost exceeds this (>= 0)")
    return ap


def parse_args(argv=None):
    ap = _parser()
    a = ap.parse_args(argv)
    if a.faces is not None and a.faces < 1:
        ap.error("--faces must be >= 1")
    if a.ratio is not None and not (math.isfinite(a.ratio) and 0 < a.ratio <= 1):
        ap.error("--ratio must be in (0, 1]")
    if a.max_error is not None and not (math.isfinite(a.max_error) and a.max_error >= 0):
        ap.error("--max_error must be a finite number >= 0")
    return a


def main(argv=None):
    a = parse_args(argv)
    v, c, f = io.read_mesh_ply(a.ply)
    target = a.faces if a.faces is not None else max(1, round(a.ratio * len(f)))
    dev = torch.device("cuda", torch.cuda.current_device())
    V, C, F, st = simplify_mesh(torch.from_numpy(np.ascontiguousarray(v)).to(dev),
                                torch.from_numpy(np.ascontiguousarray(c)).to(dev),
                                torch.from_numpy(np.ascontiguousarray(f)).to(dev), target,
                                max_error=a.max_error)
    mesh.write_mesh_ply(a.out, V, C, F)
    print(f"{a.ply}: {st['faces_in']} -> {st['faces']} faces, {st['vertices_in']} -> "
          f"{st['vertices']} vertices in {st['rounds']} rounds ({st['stop']}); wrote {a.out}")


if __name__ == "__main__":
    main()
