"""Refine a mesh against its views on the GPU: each vertex moves along its normal to where its views
agree photometrically (csrc/refine.cu; float64 numpy restatement in oracle/refine_oracle.py).

    verts, colours, faces, stats = refine_mesh(verts, colours, faces, images, Ps, sources)

    python -m casmvsnet_pl_b200.refine --ply mesh.ply --cams DIR --images DIR --pair pair.txt
                                       [--view_names FILE] [--iterations 3] --out refined.ply

Only vertex positions change; faces, colours and the vertex order do not.  The rule (stated in
full in csrc/refine.cu and include/casmvs.h), per iteration it = 0 .. T-1:
1. n_v = the normalised sum, in double and ascending face order, of (x1 - x0) x (x2 - x0) over
   v's faces; a zero sum makes v unseen;
2. v is visible in view j when it passes texturing's vertex test against the view's key buffer of
   the current mesh (w > 0, inside the PAD margin, w <= depth (1 + DEPTH_TOL) at the nearest
   pixel) and |cos(n_v, eye_j - v)| >= MIN_COS;
3. the reference is the visible view of largest |cos| (ties to the lower index); the sources are
   its pair-file sources in which v is visible, in pair order, at most S_MAX; without a reference
   or a source v is unseen;
4. along the normal, candidates k = -K .. K at delta_k = k rho STEP / 2^it (rho: the world size of
   v's reference pixel at its depth) are scored by the mean ZNCC, over the sources, of a
   (2R+1)^2 patch of grey samples spaced SPACING rho apart in the tangent plane;
5. the best valid k (ties to the smaller |k|, then the smaller k; k = 0 unless the best beats a
   valid S_0 by MIN_GAIN), refined by a parabola when k* != 0 is interior, gives d; its score is
   the confidence c when k = 0 is valid and the score is >= MIN_SCORE, else c = d = 0;
6. J Jacobi rounds d <- (c d0 + LAMBDA sum_N(v) d_u) / (c + LAMBDA |N(v)|) over the one-ring,
   then v <- v + d n.
This is a discrete sweep along the normal in the style of PMVS patch optimisation, not OpenMVS's
gradient flow: every vertex is independent and every sum has a fixed order, so two runs give the
same bits."""
from __future__ import annotations

import argparse
import ctypes
import glob
import os

import numpy as np
import torch

from . import _lib, io, mesh, texture

R = 2
K = 4
STEP = 1.0
ITERATIONS = 3
S_MAX = 4
SPACING = 4.0
MIN_GAIN = 5e-4
VAR_MIN = 1e-4
MIN_SCORE = 0.3
LAMBDA = 1.0
SMOOTH_ROUNDS = 4
PAD, MIN_COS, DEPTH_TOL, VIEW_BATCH = texture.PAD, texture.MIN_COS, texture.DEPTH_TOL, texture.VIEW_BATCH
NO_K = -1000
# device bytes per vertex: two vertex copies (24), normal (24), ref and sources (20), rho, best,
# d0, conf and two smoothing buffers (48), kstar (4), the vertex -> face and one-ring CSR pointers (8)
BYTES_PER_VERTEX = 128
# device bytes per face: the vertex -> face CSR and its sort (3 x 20), the one-ring's edge keys,
# their sort and unique (6 x 24)
BYTES_PER_FACE = 204


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _csr(rows, cols, n):
    """(ptr (n+1,) int32, cols int32) of (row, col) pairs already sorted by row."""
    ptr = torch.zeros(n + 1, dtype=torch.int32, device=rows.device)
    ptr[1:] = torch.cumsum(torch.bincount(rows, minlength=n), 0)
    return ptr, cols.int().contiguous()


def topology(faces, V):
    """-> (vf_ptr, vf_face): each vertex's faces ascending; (nb_ptr, nb_ids): its one-ring over
    the mesh's edges, ascending.  All int32 on the faces' device."""
    f = faces.long()
    F = len(f)
    corner_v = f.reshape(-1)
    order = torch.sort(corner_v, stable=True).indices          # corners in face order per vertex
    vf = _csr(corner_v[order], order // 3, V)
    a, b = f.reshape(-1), f.roll(-1, 1).reshape(-1)
    key = torch.cat([(a << 32) | b, (b << 32) | a])
    key = torch.unique(key[(a != b).repeat(2)], sorted=True)
    nb = _csr(key >> 32, key & 0xFFFFFFFF, V)
    return vf, nb


def source_csr(sources, n_views, device):
    """Pair-file sources per view (lists of view indices) -> (src_ptr, src_ids) int32."""
    ptr = np.zeros(n_views + 1, np.int32)
    ptr[1:] = np.cumsum([len(s) for s in sources])
    ids = np.array([j for s in sources for j in s] or [0], np.int32)
    return torch.from_numpy(ptr).to(device), torch.from_numpy(ids).to(device)


def grey_images(images):
    """Each view's grey image (H,W) float64, ((0.299 R + 0.587 G) + 0.114 B) / 255."""
    lib, out = _lib.load(), []
    for im in images:
        g = torch.empty(im.shape[:2], dtype=torch.float64, device=im.device)
        _lib.check(lib.casmvs_refine_grey(_ptr(im), g.numel(), _ptr(g), _stream()), "refine_grey")
        out.append(g)
    return out


def normals(verts, faces, vf):
    """Step 1 -> normal (V,3) float64, 0 for an unseen vertex."""
    V = len(verts)
    n = torch.empty(V, 3, dtype=torch.float64, device=verts.device)
    _lib.check(_lib.load().casmvs_refine_normals(_ptr(verts), V, _ptr(faces), _ptr(vf[0]), _ptr(vf[1]),
                                                 _ptr(n), _stream()), "refine_normals")
    return n


def visibility(verts, faces, normal, images, Ps, eyes, batch=VIEW_BATCH):
    """Step 2 -> vis (V, words) int32 bitset, bit j of word j // 32 for view j, one batch of key
    buffers alive at a time."""
    lib = _lib.load()
    V, F, dev = len(verts), len(faces), verts.device
    words = max(1, (len(images) + 31) // 32)
    vis = torch.zeros(V, words, dtype=torch.int32, device=dev)
    ws_bytes = lib.casmvs_render_mesh_workspace_bytes(F)
    for b in range(0, len(images), batch):
        ids = list(range(b, min(b + batch, len(images))))
        zb, wss = [], []
        for v in ids:
            H, W = images[v].shape[:2]
            zb.append(torch.empty(H * W, dtype=torch.int64, device=dev))
            wss.append(torch.empty((ws_bytes + 3) // 4, dtype=torch.int32, device=dev))
            _lib.check(lib.casmvs_render_mesh_keys(
                _ptr(verts), V, _ptr(faces), F, Ps[v].ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                W, H, _ptr(zb[-1]), _ptr(wss[-1]), wss[-1].numel() * 4, _stream()), "render_mesh_keys")
        P = np.ascontiguousarray(np.stack([Ps[v] for v in ids]), np.float32)
        eye = np.ascontiguousarray(eyes[ids], np.float64)
        wh = np.array([[images[v].shape[1], images[v].shape[0]] for v in ids], np.int32)
        vi = np.array(ids, np.int32)
        ptrs = (ctypes.c_void_p * len(ids))(*[z.data_ptr() for z in zb])
        _lib.check(lib.casmvs_refine_visibility(
            _ptr(verts), _ptr(normal), V, len(ids), P.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
            eye.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
            wh.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
            vi.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), ptrs, _ptr(vis), words, _stream()),
            "refine_visibility")
        del zb, wss
    return vis


def select(verts, normal, vis, eyes_dev, src_csr):
    """Step 3 -> (ref (V,) int32, -1 = unseen; src (V, S_MAX) int32, -1 past the last)."""
    V = len(verts)
    ref = torch.empty(V, dtype=torch.int32, device=verts.device)
    src = torch.empty(V, S_MAX, dtype=torch.int32, device=verts.device)
    _lib.check(_lib.load().casmvs_refine_select(
        _ptr(verts), _ptr(normal), V, _ptr(vis), vis.shape[1], len(eyes_dev), _ptr(eyes_dev),
        _ptr(src_csr[0]), _ptr(src_csr[1]), _ptr(ref), _ptr(src), _stream()), "refine_select")
    return ref, src


def sweep(verts, normal, ref, src, views, iteration, want_scores=False):
    """Steps 4-5 -> dict of (V,) tensors rho, best (S_k*, NaN without a valid k), kstar (NO_K
    without one), d0, conf, and with want_scores sk (V, 2K+1) float64 (NaN where k is invalid).
    `views` is the (Ps, Pinv, grey pointers, wh) device tuple of _device_views."""
    V, dev = len(verts), verts.device
    f64 = dict(dtype=torch.float64, device=dev)
    out = dict(rho=torch.empty(V, **f64), best=torch.empty(V, **f64),
               kstar=torch.empty(V, dtype=torch.int32, device=dev), d0=torch.empty(V, **f64),
               conf=torch.empty(V, **f64))
    if want_scores:
        out["sk"] = torch.empty(V, 2 * K + 1, **f64)
    Pdev, Pinv, gptr, whd = views
    _lib.check(_lib.load().casmvs_refine_sweep(
        _ptr(verts), _ptr(normal), V, _ptr(ref), _ptr(src), _ptr(Pdev), _ptr(Pinv), _ptr(gptr),
        _ptr(whd), iteration, _ptr(out["rho"]), _ptr(out["best"]), _ptr(out["kstar"]),
        _ptr(out["d0"]), _ptr(out["conf"]), _ptr(out.get("sk")), _stream()), "refine_sweep")
    return out


def smooth(nb, d0, conf, rounds=SMOOTH_ROUNDS):
    """Step 6's Jacobi rounds -> d (V,) float64."""
    lib = _lib.load()
    cur, nxt = d0.clone(), torch.empty_like(d0)
    for _ in range(rounds):
        _lib.check(lib.casmvs_refine_smooth(_ptr(nb[0]), _ptr(nb[1]), len(d0), _ptr(d0), _ptr(conf),
                                            _ptr(cur), _ptr(nxt), _stream()), "refine_smooth")
        cur, nxt = nxt, cur
    return cur


def apply(verts, normal, d):
    """v + d n per coordinate in double, rounded to float32."""
    out = torch.empty_like(verts)
    _lib.check(_lib.load().casmvs_refine_apply(_ptr(verts), _ptr(normal), _ptr(d), len(verts),
                                               _ptr(out), _stream()), "refine_apply")
    return out


def _device_views(images, Ps, greys):
    dev = images[0].device
    P64 = np.stack(Ps).astype(np.float64)
    Pdev = torch.from_numpy(np.stack(Ps).reshape(-1, 16)).to(dev)
    Pinv = torch.from_numpy(np.linalg.inv(P64).reshape(-1, 16)).to(dev)
    gptr = torch.tensor([g.data_ptr() for g in greys], dtype=torch.int64, device=dev)
    whd = torch.tensor([(im.shape[1], im.shape[0]) for im in images], dtype=torch.int32, device=dev)
    return Pdev, Pinv, gptr, whd


def check_sources(sources, n_views):
    """-> the sources as lists of ints; ValueError unless there is one list per view of view
    indices in 0 .. n_views - 1."""
    sources = [list(s) for s in sources]
    if len(sources) != n_views:
        raise ValueError(f"{len(sources)} source lists for {n_views} views")
    for j, s in enumerate(sources):
        for i in s:
            if not (isinstance(i, (int, np.integer)) and 0 <= i < n_views):
                raise ValueError(f"view {j} lists source {i!r} outside 0..{n_views - 1}")
    return [[int(i) for i in s] for s in sources]


def bytes_needed(V, F, wh):
    """Device bytes refine_mesh needs beyond its inputs."""
    grey = sum(W * H for W, H in wh) * 8
    words = max(1, (len(wh) + 31) // 32)
    return texture._bytes_needed(F, wh) + grey + V * (BYTES_PER_VERTEX + 4 * words) + F * BYTES_PER_FACE


def refine_mesh(verts, colours, faces, images, Ps, sources, iterations=ITERATIONS, max_bytes=None,
                log=print, mark=None):
    """Refine a mesh (verts (V,3) float32, colours (V,3) uint8, faces (F,3) int32 or int64, CUDA
    tensors) against views (images: (H,W,3) uint8 CUDA tensors; Ps: their 4x4 world -> pixel
    matrices; sources: per view, its pair-file source views as indices into images) ->
    (verts, colours, faces, stats).  Only the vertices move; colours and faces are returned as
    given (faces as int32).  stats: views, vertices, faces, iterations and per_iteration, a list
    of dicts: seen (vertices with a reference and a source), confident (c > 0), mean_score (mean
    S_k* over the seen vertices with a valid candidate), mean_move (mean |d| / rho over the
    confident vertices, d as applied).  Bad input raises ValueError before the GPU is used; work
    that would not fit in mesh.device_budget raises CasMVSError naming the bytes.  `mark(phase)`,
    when given, is called after each phase of each iteration: visibility (normals, key buffers
    and bits), selection, sweep, smoothing (the Jacobi rounds and the move)."""
    if not (isinstance(iterations, int) and not isinstance(iterations, bool) and iterations >= 1):
        raise ValueError(f"iterations must be an integer >= 1, got {iterations!r}")
    images, Ps = texture._check_inputs(verts, colours, faces, images, Ps)
    sources = check_sources(sources, len(images))
    mark = mark or (lambda phase: None)
    dev, V, F = verts.device, len(verts), len(faces)
    wh = [(im.shape[1], im.shape[0]) for im in images]
    stats = dict(views=len(images), vertices=V, faces=F, iterations=iterations, per_iteration=[])
    with torch.cuda.device(dev):
        budget = mesh.device_budget(dev, max_bytes)
        need = bytes_needed(V, F, wh)
        if need > budget:
            raise _lib.CasMVSError(
                f"refining {V} vertices and {F} faces against {len(images)} views needs {need} bytes "
                f"of device memory but {max(budget, 0)} bytes are available")
        faces = faces.int().contiguous()
        if not images or V == 0:
            return verts.clone(), colours, faces, stats
        cur = verts.contiguous()
        vf, nb = topology(faces, V)
        eyes = np.stack([texture.eye_of(P) for P in Ps])
        eyes_dev = torch.from_numpy(eyes).to(dev)
        src_csr = source_csr(sources, len(images), dev)
        greys = grey_images(images)
        views = _device_views(images, Ps, greys)
        for it in range(iterations):
            normal = normals(cur, faces, vf)
            vis = visibility(cur, faces, normal, images, Ps, eyes)
            mark("visibility")
            ref, src = select(cur, normal, vis, eyes_dev, src_csr)
            del vis
            mark("selection")
            sw = sweep(cur, normal, ref, src, views, it)
            mark("sweep")
            d = smooth(nb, sw["d0"], sw["conf"])
            cur = apply(cur, normal, d)
            mark("smoothing")
            conf = sw["conf"] > 0
            valid = ~torch.isnan(sw["best"])
            stats["per_iteration"].append(dict(
                seen=int((ref >= 0).sum()), confident=int(conf.sum()),
                mean_score=float(sw["best"][valid].mean()) if bool(valid.any()) else 0.0,
                mean_move=float((d[conf].abs() / sw["rho"][conf]).mean()) if bool(conf.any()) else 0.0))
    return cur, colours, faces, stats


def summary(st):
    return "; ".join(f"iteration {i}: {s['seen']} seen, {s['confident']} confident, mean score "
                     f"{s['mean_score']:.3f}, mean move {s['mean_move']:.3f} footprints"
                     for i, s in enumerate(st["per_iteration"]))


# ---------------------------------------------------------------------------- command line
def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Refine a triangle-mesh PLY against undistorted views "
                                             "on the GPU: move each vertex along its normal to "
                                             "where its views agree.")
    ap.add_argument("--ply", required=True, help="the mesh (binary PLY, as mesh.py, poisson.py and "
                                                 "simplify.py write)")
    ap.add_argument("--cams", required=True, help="directory of MVSNet *_cam.txt files whose "
                                                  "intrinsics are those of the images as stored")
    ap.add_argument("--images", required=True, help="directory of the undistorted images")
    ap.add_argument("--pair", required=True, help="pair.txt: each view's source views")
    ap.add_argument("--view_names", default=None,
                    help="view_names.txt pairing view ids with image names (default: sorted order)")
    ap.add_argument("--iterations", type=int, default=ITERATIONS,
                    help=f"refinement iterations, >= 1 (default {ITERATIONS})")
    ap.add_argument("--out", required=True, help="the refined PLY to write")
    a = ap.parse_args(argv)
    if a.iterations < 1:
        ap.error("--iterations must be >= 1")
    return a


def pair_sources(pair, view_ids):
    """pair.txt's (ref, [src]) entries -> per view of `view_ids` (in that order) its sources as
    indices; sources without a camera are left out, views without an entry have none."""
    index = {v: i for i, v in enumerate(view_ids)}
    sources = [[] for _ in view_ids]
    for r, ss in pair:
        if r in index:
            sources[index[r]] = [index[s] for s in ss if s in index]
    return sources


def main(argv=None):
    from PIL import Image
    a = parse_args(argv)
    paths, Ps = texture.read_views(a.cams, a.images, a.view_names)
    ids = [int(os.path.basename(c).split("_")[0])
           for c in sorted(glob.glob(os.path.join(a.cams, "*_cam.txt")))]
    sources = pair_sources(io.read_pair_file(a.pair), ids)
    v, c, f = io.read_mesh_ply(a.ply)
    dev = torch.device("cuda", torch.cuda.current_device())
    images = []
    for p in paths:
        if not os.path.isfile(p):
            raise ValueError(f"{p}: no such image")
        images.append(torch.from_numpy(np.asarray(Image.open(p).convert("RGB")).copy()).to(dev))
    verts, colours, faces, st = refine_mesh(torch.from_numpy(np.ascontiguousarray(v)).to(dev),
                                            torch.from_numpy(np.ascontiguousarray(c)).to(dev),
                                            torch.from_numpy(np.ascontiguousarray(f)).to(dev),
                                            images, Ps, sources, iterations=a.iterations)
    mesh.write_mesh_ply(a.out, verts, colours, faces)
    print(f"{a.ply}: {st['vertices']} vertices against {st['views']} views: {summary(st)}; "
          f"wrote {a.out}")


if __name__ == "__main__":
    main()
