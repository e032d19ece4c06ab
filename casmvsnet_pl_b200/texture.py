"""Texture a mesh from its views on the GPU: per-face view selection against each view's
visibility buffer, label smoothing, charts cut from the photographs, a packed atlas and a
textured OBJ (csrc/texture.cu; numpy restatement in oracle/texture_oracle.py, bit for bit).

    uv, page, atlas, stats = texture_mesh(verts, colours, faces, images, Ps)
    write_textured_obj("mesh.obj", verts, faces, uv, page, atlas)   # + mesh.mtl, mesh_<k>.png
    verts, faces, uv, page, atlas = read_textured_obj("mesh.obj")

    python -m casmvsnet_pl_b200.texture --ply mesh.ply --cams DIR --images DIR
                                        [--view_names FILE] --out mesh.obj

The rule (include/casmvs.h states every operation):
1. each view's visibility buffer is the triangle rasteriser's key buffer (render.py's raster pass)
   at the view's image size; views are taken VIEW_BATCH at a time, in index order;
2. face f is a candidate in view v when its three vertices project with w > 0 inside
   [PAD, W-1-PAD] x [PAD, H-1-PAD], |cos| between its normal and the line of sight to its
   centroid is >= MIN_COS (either winding), and the three vertices and the centroid each pass the
   depth test at their nearest pixel (w <= depth (1 + DEPTH_TOL)).  Its score is the projected
   area in pixels; each face keeps its K best (score desc, view asc);
3. a face's label is its best view (-1 without a candidate); then SMOOTH_ROUNDS Jacobi rounds:
   f takes L when >= 2 of its manifold-edge neighbours held L and L is one of f's candidates
   scoring >= 0.5 x its best;
4. charts are the components of equal labels >= 0 across manifold edges, named by their least
   face; a face of label -1 is a flat chart of its own;
5. a view chart's rectangle is [floor(min u) - PAD, ceil(max u) + PAD] x [floor(min v) - PAD,
   ceil(max v) + PAD] in its view; a flat chart is FLAT x FLAT texels;
6. rectangles are packed shelf next-fit in the order (height desc, width desc, chart asc) into
   S x S pages, S = PAGE_SIDE or the least power of two >= the largest side, up to MAX_PAGE_SIDE;
7. a view chart's texels are a byte copy of its rectangle; a flat chart is the mean of its face's
   vertex colours (rounded half to even); unused texels are 0;
8. a corner's UV is ((u - x0 + ox + 0.5) / S, 1 - (v - y0 + oy + 0.5) / S) in double, stored as
   float32; a flat face's corners sit on texel centres inside its square.

With level=True (`--level`), the seams between charts are then levelled by Waechter et al.'s
global colour adjustment (csrc/texture_level.cu; numpy restatement in
oracle/texture_level_oracle.py, bit for bit but for the solve).  UVs, pages, charts, the packing
and flat charts do not change; only the texels of view charts do:
1. seams: the edge of corner k of f is a seam when g = nbr[f][k] >= 0, both labels are >= 0 and
   slot[f] != slot[g]; open and non-manifold edges never are, and flat charts take no part;
2. unknowns: one RGB offset g per (chart, vertex) pair of a view-chart face's corner, numbered by
   the sorted key (slot << 32) | vertex;
3. seam colours: for each seam edge and each endpoint v, SEAM_SAMPLES points v + t (w - v),
   t = k / SEAM_SAMPLES, in double, are projected into both charts' views and sampled bilinearly
   (pixel centres at integer coordinates); f_(v,i) of the pair (v; i, j) is the (1 - t)-weighted
   mean of the view(i) samples over v's seam edges between i and j, summed in record order;
4. system: minimise sum_pairs (f_(v,i) + g_(v,i) - f_(v,j) - g_(v,j))^2 + SMOOTH_WEIGHT
   sum over each chart's unique edges (g_a - g_b)^2 + EPS sum g^2, one CSR matrix for the three
   channels.  SMOOTH_WEIGHT = 10 is Waechter's 1/lambda with lambda = 0.1.  EPS = 1e-4 only makes
   the matrix definite: the right-hand side sums to zero over every group of charts joined by
   seams, so the near-null modes it would otherwise leave carry no load.  Its damping of a chart's
   mean offset is 1 / (1 + EPS N / (2 m)) for two charts of N unknowns each meeting at m seam
   pairs: 5e-5 in the two-quad test, 0.25 % for N = 10^4 and m = 200;
5. solve: Jacobi-preconditioned conjugate gradients in double, the three channels sharing each
   SpMV, until every channel has ||r|| / ||b|| <= CG_TOL or after CG_MAX_ITERS iterations (an
   unconverged solve is logged and recorded).  The host reads the convergence flag every
   CG_CHECK_EVERY iterations; the device stops on the exact iteration either way;
6. texel offsets: each texel of a view chart sits at view pixel (x0 + k, y0 + l); its owner is the
   chart face whose projected triangle lies nearest that point, within REACH = 1.5 texels (>= sqrt 2,
   so every bilinear tap of a point inside a face is reached and sliver faces that hold no texel
   centre are still covered), ties to the lower face; its offset is the owner's corner offsets
   interpolated at the barycentrics of the nearest point;
7. apply: texel = clamp(rint(byte + offset), 0, 255) per channel; texels without an owner keep
   their bytes."""
from __future__ import annotations

import argparse
import ctypes
import glob
import os

import numpy as np
import torch

from . import _lib, io, mesh

K = 4
PAD = 2
MIN_COS = 0.1
DEPTH_TOL = 0.01
SMOOTH_ROUNDS = 4
VIEW_BATCH = 8
PAGE_SIDE = 4096
MAX_PAGE_SIDE = 16384
FLAT = 4
# device bytes per face besides the key buffers and the pages: the candidates (32), the corner
# keys, unique edges and sorts of the neighbour table (~120), labels, components, rectangles,
# slots, UVs and pages (~72)
BYTES_PER_FACE = 224
SEAM_SAMPLES = 8
SMOOTH_WEIGHT = 10.0
LEVEL_EPS = 1e-4
REACH = 1.5
CG_TOL = 1e-9
CG_MAX_ITERS = 10000
CG_CHECK_EVERY = 16
# device bytes per face of the levelling, at most 3 unknowns, 3 seam records and 15 matrix entries
# per face: corner keys and unknowns (~60), edge keys and seam records with their sorts and
# colours (~300), matrix keys, their sort and the CSR (~360), CG vectors (6 x 3 unknowns x 24 = 432)
LEVEL_BYTES_PER_FACE = 1152


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def eye_of(P):
    """The camera centre of a world -> pixel matrix (float32 P, solved in float64), float64."""
    P = np.asarray(P, np.float32).astype(np.float64)
    return -np.linalg.solve(P[:3, :3], P[:3, 3])


def neighbours(faces):
    """(F,3) int32: the face across the edge of corner k (faces[f][k] -- faces[f][(k+1)%3]) when
    exactly two distinct faces share that edge, else -1."""
    f = faces.long()
    F = len(f)
    nbr = torch.full((3 * F,), -1, dtype=torch.int32, device=f.device)
    if F == 0:
        return nbr.view(0, 3)
    g = f.roll(-1, 1)
    key = ((torch.minimum(f, g) << 32) | torch.maximum(f, g)).reshape(-1)
    _, inv, cnt = torch.unique(key, sorted=True, return_inverse=True, return_counts=True)
    order = torch.sort(inv, stable=True).indices
    start = torch.cumsum(cnt, 0) - cnt
    two = torch.nonzero(cnt == 2).squeeze(1)
    c0, c1 = order[start[two]], order[start[two] + 1]
    ok = (c0 // 3) != (c1 // 3)
    c0, c1 = c0[ok], c1[ok]
    nbr[c0] = (c1 // 3).int()
    nbr[c1] = (c0 // 3).int()
    return nbr.view(F, 3)


def _check_inputs(verts, colours, faces, images, Ps):
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
    if 3 * max(len(verts), len(faces)) >= 2 ** 31:
        raise ValueError(f"a mesh of {len(verts)} vertices and {len(faces)} faces is too large")
    if len(verts) and not bool(torch.isfinite(verts).all()):
        raise ValueError("verts holds a non-finite coordinate")
    if len(faces) and not bool(((faces >= 0) & (faces < len(verts))).all()):
        raise ValueError(f"faces holds an index outside 0..{len(verts) - 1}")
    images, Ps = list(images), list(Ps)
    if len(images) != len(Ps):
        raise ValueError(f"{len(images)} images but {len(Ps)} projection matrices")
    for i, im in enumerate(images):
        if not (torch.is_tensor(im) and im.is_cuda and im.dtype == torch.uint8 and im.dim() == 3
                and im.shape[2] == 3 and im.device == verts.device):
            raise ValueError(f"image {i} must be an (H, W, 3) uint8 CUDA tensor on the mesh's device")
        H, W = im.shape[:2]
        if not (2 * PAD < W <= MAX_PAGE_SIDE and 2 * PAD < H <= MAX_PAGE_SIDE):
            raise ValueError(f"image {i} is {W}x{H}; each side must lie in {2 * PAD + 1}.."
                             f"{MAX_PAGE_SIDE}")
    out = []
    for i, P in enumerate(Ps):
        P = np.asarray(P.cpu() if torch.is_tensor(P) else P, dtype=np.float64)
        if P.shape != (4, 4) or not np.isfinite(P).all():
            raise ValueError(f"P {i} must be a finite 4x4 world -> pixel matrix")
        out.append(np.ascontiguousarray(P, np.float32))
    return [im.contiguous() for im in images], out


def _bytes_needed(F, wh, batch=VIEW_BATCH):
    keys = max((sum(W * H for W, H in wh[b:b + batch]) for b in range(0, len(wh), batch)),
               default=0)
    ws = min(len(wh), batch) * (F + 2) * 4
    return keys * 8 + ws + F * BYTES_PER_FACE


def candidates(verts, faces, images, Ps, batch=VIEW_BATCH, mark=None):
    """Steps 1-2 -> (cand_score (F,K) float32, cand_view (F,K) int32, -1 = empty).  `mark`, when
    given, is called with "keys" after each batch's key buffers and "scores" after its scores."""
    mark = mark or (lambda phase: None)
    lib = _lib.load()
    F, dev = len(faces), verts.device
    score = torch.zeros(F, K, dtype=torch.float32, device=dev)
    view = torch.full((F, K), -1, dtype=torch.int32, device=dev)
    ws_bytes = lib.casmvs_render_mesh_workspace_bytes(F)
    for b in range(0, len(images), batch):
        ids = list(range(b, min(b + batch, len(images))))
        n = len(ids)
        zb, wss = [], []
        for v in ids:
            H, W = images[v].shape[:2]
            zb.append(torch.empty(H * W, dtype=torch.int64, device=dev))
            wss.append(torch.empty((ws_bytes + 3) // 4, dtype=torch.int32, device=dev))
            _lib.check(lib.casmvs_render_mesh_keys(
                _ptr(verts), len(verts), _ptr(faces), F, Ps[v].ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                W, H, _ptr(zb[-1]), _ptr(wss[-1]), wss[-1].numel() * 4, _stream()), "render_mesh_keys")
        mark("keys")
        P = np.ascontiguousarray(np.stack([Ps[v] for v in ids]), np.float32)
        eye = np.ascontiguousarray(np.stack([eye_of(Ps[v]) for v in ids]), np.float64)
        wh = np.array([[images[v].shape[1], images[v].shape[0]] for v in ids], np.int32)
        vi = np.array(ids, np.int32)
        ptrs = (ctypes.c_void_p * n)(*[z.data_ptr() for z in zb])
        _lib.check(lib.casmvs_texture_scores(
            _ptr(verts), _ptr(faces), F, n, P.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
            eye.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
            wh.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
            vi.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), ptrs, _ptr(score), _ptr(view),
            _stream()), "texture_scores")
        mark("scores")
        del zb, wss
    return score, view


def smooth(nbr, score, view, labels, rounds=SMOOTH_ROUNDS):
    """Step 3's Jacobi rounds -> the labels after `rounds` rounds."""
    lib = _lib.load()
    cur = labels.clone()
    nxt = torch.empty_like(cur)
    for _ in range(rounds):
        _lib.check(lib.casmvs_texture_smooth(_ptr(nbr), _ptr(score), _ptr(view), len(cur), _ptr(cur),
                                             _ptr(nxt), _stream()), "texture_smooth")
        cur, nxt = nxt, cur
    return cur


def components(nbr, labels):
    """Step 4 -> (comp (F,) int32, the least face of each face's chart; hook rounds)."""
    F = len(labels)
    comp = torch.empty(F, dtype=torch.int32, device=labels.device)
    flag = torch.empty(1, dtype=torch.int32, device=labels.device)
    rounds = ctypes.c_int(0)
    _lib.check(_lib.load().casmvs_texture_charts(_ptr(nbr), _ptr(labels), F, _ptr(comp), _ptr(flag),
                                                 ctypes.byref(rounds), _stream()), "texture_charts")
    return comp, rounds.value


def chart_table(verts, faces, labels, comp, Pdev):
    """Step 5 -> (roots (C,) int64 ascending, charts (C,9) int32 numpy with the page columns 0)."""
    F = len(faces)
    rect = torch.empty(F, 4, dtype=torch.int32, device=verts.device)
    _lib.check(_lib.load().casmvs_texture_rects(_ptr(verts), _ptr(faces), F, _ptr(labels), _ptr(comp),
                                                _ptr(Pdev), _ptr(rect), _stream()), "texture_rects")
    roots = torch.nonzero(comp == torch.arange(F, dtype=torch.int32, device=comp.device)).squeeze(1)
    lab, r = labels[roots], rect[roots]
    flat = (lab < 0).unsqueeze(1)
    box = torch.where(flat, torch.tensor([0, 0, FLAT - 1, FLAT - 1], dtype=torch.int32,
                                         device=r.device), r)
    charts = torch.cat([roots.int().unsqueeze(1), lab.unsqueeze(1), box,
                        torch.zeros(len(roots), 3, dtype=torch.int32, device=r.device)], 1)
    return roots, charts.cpu().numpy()


def page_side(w, h):
    """Step 6's page side for rectangles of widths w and heights h; ValueError above the limit."""
    side = int(max(np.max(w, initial=0), np.max(h, initial=0)))
    if side > MAX_PAGE_SIDE:
        raise ValueError(f"a chart of {side} texels per side does not fit a page of at most "
                         f"{MAX_PAGE_SIDE}")
    S = PAGE_SIDE
    while S < side:
        S *= 2
    return S


def pack(ids, w, h, S):
    """Shelf next-fit in the order (height desc, width desc, id asc) -> (page, ox, oy) int32
    arrays aligned with the inputs, and the number of pages."""
    ids, w, h = (np.asarray(a, np.int64) for a in (ids, w, h))
    order = np.lexsort((ids, -w, -h))
    page = np.zeros(len(ids), np.int32)
    ox, oy = np.zeros(len(ids), np.int32), np.zeros(len(ids), np.int32)
    p = x = y = shelf = 0
    for i, ww, hh in zip(order.tolist(), w[order].tolist(), h[order].tolist()):
        if x + ww > S:
            x, y, shelf = 0, y + shelf, 0
        if y + hh > S:
            p, x, y, shelf = p + 1, 0, 0, 0
        page[i], ox[i], oy[i] = p, x, y
        x += ww
        shelf = max(shelf, hh)
    return page, ox, oy, (p + 1 if len(ids) else 0)


# ---------------------------------------------------------------------------- seam levelling
def _i64(x):
    return torch.as_tensor(x, dtype=torch.int64)


def level_unknowns(faces, labels, slot):
    """Levelling step 2 -> (unknowns (n,) int64 ascending, (slot << 32) | vertex of every corner
    of a view-chart face; corner (F,3) int32, the unknown of each corner, -1 on flat faces)."""
    lib, F = _lib.load(), len(faces)
    keys = torch.empty(3 * F, dtype=torch.int64, device=faces.device)
    _lib.check(lib.casmvs_texture_level_keys(_ptr(faces), F, _ptr(labels), _ptr(slot), _ptr(keys),
                                             _stream()), "texture_level_keys")
    unk = torch.unique(keys[keys >= 0], sorted=True)
    corner = torch.empty(F, 3, dtype=torch.int32, device=faces.device)
    _lib.check(lib.casmvs_texture_level_corners(_ptr(keys), F, _ptr(unk), len(unk), _ptr(corner),
                                                _stream()), "texture_level_corners")
    return unk, corner


def level_edges(nbr, faces, labels, slot, corner):
    """Levelling step 1 -> (rec_key, rec_sub) of the seam endpoint records, sorted by (pair key,
    record), and the distinct smoothing-edge keys (min << 32) | max of unknowns, ascending."""
    lib, F = _lib.load(), len(faces)
    rec = torch.empty(6 * F, dtype=torch.int64, device=faces.device)
    sm = torch.empty(3 * F, dtype=torch.int64, device=faces.device)
    _lib.check(lib.casmvs_texture_level_edges(_ptr(nbr), _ptr(faces), F, _ptr(labels), _ptr(slot),
                                              _ptr(corner), _ptr(rec), _ptr(sm), _stream()),
               "texture_level_edges")
    sub = torch.nonzero(rec >= 0).squeeze(1)
    key, order = torch.sort(rec[sub], stable=True)
    return key, sub[order].contiguous(), torch.unique(sm[sm >= 0], sorted=True)


def level_seam_colours(verts, faces, labels, slot, nbr, rec_key, rec_sub, img_ptrs, img_wh, Pdev):
    """Levelling step 3 -> (pair keys (P,) int64 ascending, (a << 32) | b; fpair (P,6) float64,
    f_a and f_b: the seam colours of each pair in the lower and the upper chart's view)."""
    lib, R = _lib.load(), len(rec_sub)
    rec = torch.empty(R, 6, dtype=torch.float64, device=verts.device)
    _lib.check(lib.casmvs_texture_level_samples(_ptr(verts), _ptr(faces), _ptr(labels), _ptr(slot),
                                                _ptr(nbr), _ptr(rec_sub), R, _ptr(Pdev),
                                                _ptr(img_ptrs), _ptr(img_wh), _ptr(rec), _stream()),
               "texture_level_samples")
    keys, cnt = torch.unique_consecutive(rec_key, return_counts=True)
    seg = torch.zeros(len(keys) + 1, dtype=torch.int64, device=verts.device)
    seg[1:] = torch.cumsum(cnt, 0)
    fpair = torch.empty(len(keys), 6, dtype=torch.float64, device=verts.device)
    _lib.check(lib.casmvs_texture_level_pairs(_ptr(rec), _ptr(seg), len(keys), _ptr(fpair),
                                              _stream()), "texture_level_pairs")
    return keys, fpair


def level_system(pair_keys, smooth_keys, n, fpair):
    """Levelling step 4 -> (rowptr (n+1) int32, col (nnz) int32, val (nnz), diag (n), rhs (n,3)
    float64): A g = rhs, A in CSR with columns ascending in each row."""
    dev = fpair.device
    lo32 = 0xFFFFFFFF
    lp, hp, ls, hs = pair_keys >> 32, pair_keys & lo32, smooth_keys >> 32, smooth_keys & lo32
    a = torch.arange(n, dtype=torch.int64, device=dev)
    P, E = len(pair_keys), len(smooth_keys)
    ekey = torch.cat([(lp << 32) | hp, (hp << 32) | lp, (ls << 32) | hs, (hs << 32) | ls,
                      (a << 32) | a])
    pid = torch.arange(P, dtype=torch.int32, device=dev)
    etype = torch.cat([pid, pid, torch.full((2 * E,), -2, dtype=torch.int32, device=dev),
                       torch.full((n,), -1, dtype=torch.int32, device=dev)])
    ekey, order = torch.sort(ekey)
    etype = etype[order].contiguous()
    del order
    nnz = len(ekey)
    rowptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
    col = torch.empty(nnz, dtype=torch.int32, device=dev)
    val = torch.empty(nnz, dtype=torch.float64, device=dev)
    diag = torch.empty(n, dtype=torch.float64, device=dev)
    rhs = torch.empty(n, 3, dtype=torch.float64, device=dev)
    _lib.check(_lib.load().casmvs_texture_level_system(
        _ptr(ekey), _ptr(etype), nnz, n, _ptr(fpair), _ptr(rowptr), _ptr(col), _ptr(val), _ptr(diag),
        _ptr(rhs), _stream()), "texture_level_system")
    return rowptr, col, val, diag, rhs


def level_solve(rowptr, col, val, diag, rhs, tol=CG_TOL, max_iters=CG_MAX_ITERS,
                check_every=CG_CHECK_EVERY):
    """Levelling step 5 -> (g (n,3) float64, iterations, ratios (3 floats), converged)."""
    lib, n = _lib.load(), len(diag)
    g = torch.empty(n, 3, dtype=torch.float64, device=rhs.device)
    ws = torch.empty(max(1, lib.casmvs_texture_level_cg_workspace_bytes(n)), dtype=torch.uint8,
                     device=rhs.device)
    iters, conv = ctypes.c_int(0), ctypes.c_int(0)
    ratios = (ctypes.c_double * 3)()
    _lib.check(lib.casmvs_texture_level_cg(
        _ptr(rowptr), _ptr(col), _ptr(val), _ptr(diag), _ptr(rhs), n, _ptr(g), _ptr(ws), ws.numel(),
        max_iters, tol, check_every, ctypes.byref(iters), ratios, ctypes.byref(conv), _stream()),
        "texture_level_cg")
    return g, iters.value, list(ratios), bool(conv.value)


def level_owners(verts, faces, labels, slot, cdev, Pdev, S, n_pages):
    """Levelling step 6 -> owner (pages,S,S) int64: (f32 distance bits << 32) | face of each
    texel's owner, -1 (all bits set) where it has none."""
    owner = torch.full((n_pages, S, S), -1, dtype=torch.int64, device=verts.device)
    _lib.check(_lib.load().casmvs_texture_level_owners(
        _ptr(verts), _ptr(faces), len(faces), _ptr(labels), _ptr(slot), _ptr(cdev), _ptr(Pdev), S,
        _ptr(owner), _stream()), "texture_level_owners")
    return owner


def level_apply(owner, verts, faces, labels, slot, cdev, Pdev, corner, g, atlas):
    """Levelling step 7, in place on atlas (pages,S,S,3) uint8."""
    _lib.check(_lib.load().casmvs_texture_level_apply(
        _ptr(owner), owner.numel(), _ptr(verts), _ptr(faces), _ptr(labels), _ptr(slot), _ptr(cdev),
        _ptr(Pdev), atlas.shape[1], _ptr(corner), _ptr(g), _ptr(atlas), _stream()),
        "texture_level_apply")


def seam_rms(fpair, g=None, pair_keys=None):
    """RMS over seam pairs and channels of f_a - f_b, or with g of f_a + g_a - f_b - g_b."""
    if not len(fpair):
        return 0.0
    d = fpair[:, :3] - fpair[:, 3:]
    if g is not None:
        d = d + g[pair_keys >> 32] - g[pair_keys & 0xFFFFFFFF]
    return float(torch.sqrt((d * d).mean()))


def level_seams(verts, faces, labels, slot, cdev, Pdev, img_ptrs, img_wh, nbr, atlas, mark=None,
                log=print):
    """Steps 1-7 of the seam levelling on texture_mesh's state, atlas changed in place -> the
    stats of texture_mesh's stats["level"].  `mark(phase)` after seams, assembly, solve, apply."""
    mark = mark or (lambda phase: None)
    unk, corner = level_unknowns(faces, labels, slot)
    rec_key, rec_sub, smooth_keys = level_edges(nbr, faces, labels, slot, corner)
    pair_keys, fpair = level_seam_colours(verts, faces, labels, slot, nbr, rec_key, rec_sub,
                                          img_ptrs, img_wh, Pdev)
    n_records = len(rec_sub)
    del rec_key, rec_sub
    mark("seams")
    rowptr, col, val, diag, rhs = level_system(pair_keys, smooth_keys, len(unk), fpair)
    mark("assembly")
    g, iters, ratios, converged = level_solve(rowptr, col, val, diag, rhs)
    nnz = len(col)
    del rowptr, col, val, diag, rhs
    mark("solve")
    if not converged:
        log(f"texture level: conjugate gradients stopped after {iters} iterations with relative "
            f"residuals {', '.join(f'{r:.3g}' for r in ratios)} above {CG_TOL:g}")
    pages, S = atlas.shape[0], atlas.shape[1]
    owner = level_owners(verts, faces, labels, slot, cdev, Pdev, S, pages)
    level_apply(owner, verts, faces, labels, slot, cdev, Pdev, corner, g, atlas)
    adjusted = int((owner != -1).sum())
    mark("apply")
    return dict(unknowns=len(unk), seam_pairs=len(pair_keys), seam_records=n_records,
                smoothing_edges=len(smooth_keys), nnz=nnz, texels_adjusted=adjusted,
                cg_iterations=iters, cg_ratios=ratios, converged=converged,
                seam_rms_before=seam_rms(fpair), seam_rms_after=seam_rms(fpair, g, pair_keys))


def texture_mesh(verts, colours, faces, images, Ps, rounds=SMOOTH_ROUNDS, max_bytes=None,
                 mark=None, level=False, log=print):
    """Texture a mesh (verts (N,3) float32, colours (N,3) uint8, faces (M,3) int32 or int64, CUDA
    tensors) from views (images: (H,W,3) uint8 CUDA tensors; Ps: 4x4 world -> pixel matrices of
    those images) -> (uv (M,3,2) float32 per corner, page (M,) int32, atlas (pages,S,S,3) uint8,
    stats: views, faces, candidates_per_face, unseen_faces, charts_unsmoothed, charts,
    flat_charts, pages, page_side, packed_share, hook_rounds), all on the mesh's device.  With no
    views every face is flat.  Bad input raises ValueError before the GPU is used; work that
    would not fit in mesh.device_budget raises CasMVSError naming the bytes.  `mark(phase)`, when
    given, is called after each phase: keys and scores (once per batch of views), smooth, charts,
    pack, fill, and with `level` seams, assembly, solve, apply.  `level` levels the seams after
    the fill (the module docstring's second rule) and adds stats["level"]: unknowns, seam_pairs,
    seam_records, smoothing_edges, nnz, texels_adjusted, cg_iterations, cg_ratios, converged,
    seam_rms_before, seam_rms_after; an unconverged solve is reported through `log`."""
    images, Ps = _check_inputs(verts, colours, faces, images, Ps)
    if not (isinstance(rounds, int) and rounds >= 0):
        raise ValueError(f"rounds must be an integer >= 0, got {rounds!r}")
    mark = mark or (lambda phase: None)
    dev, F = verts.device, len(faces)
    wh = [(im.shape[1], im.shape[0]) for im in images]
    lib = _lib.load()
    with torch.cuda.device(dev):
        budget = mesh.device_budget(dev, max_bytes)
        need = _bytes_needed(F, wh) + (F * LEVEL_BYTES_PER_FACE if level else 0)
        if need > budget:
            raise _lib.CasMVSError(
                f"texturing {F} faces from {len(images)} views needs {need} bytes of device memory "
                f"but {max(budget, 0)} bytes are available")
        verts, colours = verts.contiguous(), colours.contiguous()
        faces = faces.int().contiguous()
        score, view = candidates(verts, faces, images, Ps, mark=mark)
        nbr = neighbours(faces)
        labels0 = view[:, 0].contiguous()
        labels = smooth(nbr, score, view, labels0, rounds)
        mark("smooth")
        comp0, _ = components(nbr, labels0)
        comp, hook_rounds = components(nbr, labels)
        Pdev = torch.from_numpy(np.stack(Ps).reshape(-1, 16) if Ps else np.zeros((1, 16), np.float32)
                                ).to(dev)
        roots, charts = chart_table(verts, faces, labels, comp, Pdev)
        mark("charts")
        w, h = charts[:, 4] - charts[:, 2] + 1, charts[:, 5] - charts[:, 3] + 1
        S = page_side(w, h)
        charts[:, 6], charts[:, 7], charts[:, 8], n_pages = pack(charts[:, 0], w, h, S)
        mark("pack")
        page_bytes = n_pages * S * S * (3 + (8 if level else 0))
        budget = mesh.device_budget(dev, max_bytes if max_bytes is None else max_bytes - need)
        if page_bytes > budget:
            raise _lib.CasMVSError(
                f"the atlas of {n_pages} pages of {S}x{S} needs {page_bytes} bytes of device "
                f"memory but {max(budget, 0)} bytes are available")
        cdev = torch.from_numpy(np.ascontiguousarray(charts)).to(dev)
        atlas = torch.zeros(n_pages, S, S, 3, dtype=torch.uint8, device=dev)
        img_ptrs = torch.tensor([im.data_ptr() for im in images] or [0], dtype=torch.int64, device=dev)
        img_wh = torch.tensor(wh or [(0, 0)], dtype=torch.int32, device=dev)
        _lib.check(lib.casmvs_texture_fill(_ptr(cdev), len(charts), _ptr(img_ptrs), _ptr(img_wh),
                                           _ptr(colours), _ptr(faces), S, _ptr(atlas), _stream()),
                   "texture_fill")
        slot = torch.searchsorted(roots.int(), comp).int()
        uv = torch.empty(F, 3, 2, dtype=torch.float32, device=dev)
        page = torch.empty(F, dtype=torch.int32, device=dev)
        _lib.check(lib.casmvs_texture_uvs(_ptr(verts), _ptr(faces), F, _ptr(labels), _ptr(slot),
                                          _ptr(cdev), _ptr(Pdev), S, _ptr(uv), _ptr(page), _stream()),
                   "texture_uvs")
        mark("fill")
        if level:
            level_stats = level_seams(verts, faces, labels, slot, cdev, Pdev, img_ptrs, img_wh, nbr,
                                      atlas, mark, log)
        n_cand = (view >= 0).sum(1)
        stats = dict(views=len(images), faces=F,
                     candidates_per_face=float(n_cand.float().mean()) if F else 0.0,
                     unseen_faces=int((n_cand == 0).sum()),
                     charts_unsmoothed=int((comp0 == torch.arange(F, device=dev)).sum()),
                     charts=len(charts), flat_charts=int((charts[:, 1] < 0).sum()),
                     pages=n_pages, page_side=S,
                     packed_share=float((w.astype(np.int64) * h).sum() / (n_pages * S * S))
                     if n_pages else 0.0,
                     hook_rounds=hook_rounds)
        if level:
            stats["level"] = level_stats
    return uv, page, atlas, stats


# ---------------------------------------------------------------------------- files
def _host(t, dt):
    return np.ascontiguousarray(t.cpu().numpy() if torch.is_tensor(t) else np.asarray(t), dt)


def write_textured_obj(path, verts, faces, uv, page, atlas):
    """Write <name>.obj, <name>.mtl and <name>_<k>.png (one per atlas page).  The OBJ holds one
    `v` per vertex, one `vt` per face corner (corner k of face f is vt 3f + k + 1) and the faces
    grouped by page (stable) under `usemtl page_<k>`; the MTL maps page_<k> to its PNG.
    -> the paths written."""
    from PIL import Image
    path = str(path)
    if not path.endswith(".obj"):
        raise ValueError(f"{path}: the mesh path must end in .obj")
    base = path[:-4]
    name = os.path.basename(base)
    V, Fc = _host(verts, np.float32).reshape(-1, 3), _host(faces, np.int64).reshape(-1, 3)
    UV, pg = _host(uv, np.float32).reshape(-1, 2), _host(page, np.int64).reshape(-1)
    A = _host(atlas, np.uint8)
    if not (len(UV) == 3 * len(Fc) and len(pg) == len(Fc)):
        raise ValueError("uv must hold 3 corners and page one entry per face")
    if len(pg) and (pg.min() < 0 or pg.max() >= len(A)):
        raise ValueError("a face's page lies outside the atlas")
    order = np.argsort(pg, kind="stable")
    parts = [f"mtllib {name}.mtl\n",
             ("v %.9g %.9g %.9g\n" * len(V)) % tuple(V.astype(np.float64).ravel().tolist()),
             ("vt %.9g %.9g\n" * len(UV)) % tuple(UV.astype(np.float64).ravel().tolist())]
    for k in range(len(A)):
        sel = order[pg[order] == k]
        if not len(sel):
            continue
        vi = Fc[sel] + 1
        ti = 3 * sel[:, None] + np.arange(1, 4)
        parts.append(f"usemtl page_{k}\n")
        parts.append(("f %d/%d %d/%d %d/%d\n" * len(sel)) %
                     tuple(np.stack([vi, ti], 2).ravel().tolist()))
    with open(path, "w") as f:
        f.write("".join(parts))
    out = [path, base + ".mtl"]
    with open(out[1], "w") as f:
        f.write("".join(f"newmtl page_{k}\nKa 1 1 1\nKd 1 1 1\nKs 0 0 0\nillum 1\n"
                        f"map_Kd {name}_{k}.png\n\n" for k in range(len(A))))
    for k in range(len(A)):
        out.append(f"{base}_{k}.png")
        Image.fromarray(A[k]).save(out[-1], compress_level=1)
    return out


def read_textured_obj(path):
    """-> (verts (N,3) float32, faces (M,3) int32, uv (M,3,2) float32, page (M,) int32,
    atlas (pages,S,S,3) uint8) of a file write_textured_obj wrote, faces in their original order."""
    from PIL import Image
    path = str(path)
    d = os.path.dirname(path)
    with open(path) as f:
        lines = f.read().splitlines()
    mtl, v, vt, fv, ft, fp = None, [], [], [], [], []
    pages, cur = {}, None
    for ln in lines:
        tok = ln.split()
        if not tok:
            continue
        if tok[0] == "mtllib":
            mtl = tok[1]
        elif tok[0] == "v":
            v.append(tok[1:4])
        elif tok[0] == "vt":
            vt.append(tok[1:3])
        elif tok[0] == "usemtl":
            cur = int(tok[1].rsplit("_", 1)[1])
        elif tok[0] == "f":
            a = [t.split("/") for t in tok[1:4]]
            fv.append([int(x[0]) - 1 for x in a])
            ft.append([int(x[1]) - 1 for x in a])
            fp.append(cur)
    if mtl is None:
        raise ValueError(f"{path}: no mtllib")
    with open(os.path.join(d, mtl)) as f:
        name = None
        for ln in f.read().splitlines():
            tok = ln.split()
            if tok and tok[0] == "newmtl":
                name = int(tok[1].rsplit("_", 1)[1])
            elif tok and tok[0] == "map_Kd":
                pages[name] = np.asarray(Image.open(os.path.join(d, tok[1])).convert("RGB"))
    verts = np.array(v, np.float32).reshape(-1, 3)
    uvs = np.array(vt, np.float32).reshape(-1, 2)
    fv, ft = np.array(fv, np.int64).reshape(-1, 3), np.array(ft, np.int64).reshape(-1, 3)
    orig = ft[:, 0] // 3
    faces = np.zeros_like(fv)
    faces[orig] = fv
    page = np.zeros(len(fv), np.int32)
    page[orig] = np.array(fp, np.int32)
    atlas = (np.stack([pages[k] for k in sorted(pages)]) if pages else np.zeros((0, 1, 1, 3), np.uint8))
    return verts, faces.astype(np.int32), uvs.reshape(-1, 3, 2), page, atlas


# ---------------------------------------------------------------------------- command line
IMAGE_EXTS = (".jpg", ".jpeg", ".png", ".bmp", ".tif", ".tiff")


def read_views(cam_dir, image_dir, view_names=None):
    """-> (image paths, P (4,4) float32 matrices) of the MVSNet *_cam.txt files in cam_dir paired
    with images: by view_names.txt (`<view id> <image name>` per line, the id the camera file's
    name starts with) or, without it, by sorted order, when the counts agree."""
    cams = sorted(glob.glob(os.path.join(cam_dir, "*_cam.txt")))
    if not cams:
        raise ValueError(f"{cam_dir}: no *_cam.txt camera files")
    if view_names:
        names = {}
        with open(view_names) as f:
            for ln in f:
                if ln.strip():
                    vid, name = ln.strip().split(maxsplit=1)
                    names[int(vid)] = name
        paths = []
        for c in cams:
            vid = int(os.path.basename(c).split("_")[0])
            if vid not in names:
                raise ValueError(f"{view_names}: no image name for view {vid} ({c})")
            paths.append(os.path.join(image_dir, os.path.basename(names[vid])))
    else:
        paths = sorted(os.path.join(image_dir, n) for n in os.listdir(image_dir)
                       if n.lower().endswith(IMAGE_EXTS))
        if len(paths) != len(cams):
            raise ValueError(f"{image_dir} holds {len(paths)} images and {cam_dir} {len(cams)} "
                             "cameras: pair them with --view_names")
    Ps = []
    for c in cams:
        Kc, E, _ = io.read_cam_file(c)
        Ps.append(_projection(Kc, E))
    return paths, Ps


def _projection(Kc, E):
    K4 = np.eye(4)
    K4[:3, :3] = np.asarray(Kc, np.float64)
    return (K4 @ np.asarray(E, np.float64)).astype(np.float32)


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Texture a triangle-mesh PLY from undistorted views on "
                                             "the GPU and write a textured OBJ.")
    ap.add_argument("--ply", required=True, help="the mesh (binary PLY, as mesh.py, poisson.py and "
                                                 "simplify.py write)")
    ap.add_argument("--cams", required=True, help="directory of MVSNet *_cam.txt files whose "
                                                  "intrinsics are those of the images as stored")
    ap.add_argument("--images", required=True, help="directory of the undistorted images")
    ap.add_argument("--view_names", default=None,
                    help="view_names.txt pairing view ids with image names (default: sorted order)")
    ap.add_argument("--out", required=True, help="the OBJ to write (its .mtl and _<k>.png beside it)")
    ap.add_argument("--level", action="store_true",
                    help="level the colour seams between charts (global colour adjustment)")
    a = ap.parse_args(argv)
    if not a.out.endswith(".obj"):
        ap.error("--out must end in .obj")
    return a


def main(argv=None):
    from PIL import Image
    a = parse_args(argv)
    paths, Ps = read_views(a.cams, a.images, a.view_names)
    v, c, f = io.read_mesh_ply(a.ply)
    dev = torch.device("cuda", torch.cuda.current_device())
    images = []
    for p in paths:
        if not os.path.isfile(p):
            raise ValueError(f"{p}: no such image")
        images.append(torch.from_numpy(np.asarray(Image.open(p).convert("RGB")).copy()).to(dev))
    uv, page, atlas, st = texture_mesh(torch.from_numpy(np.ascontiguousarray(v)).to(dev),
                                       torch.from_numpy(np.ascontiguousarray(c)).to(dev),
                                       torch.from_numpy(np.ascontiguousarray(f)).to(dev), images, Ps,
                                       level=a.level)
    write_textured_obj(a.out, v, f, uv, page, atlas)
    print(f"{a.ply}: {st['faces']} faces from {st['views']} views, {st['unseen_faces']} unseen, "
          f"{st['charts']} charts on {st['pages']} pages of {st['page_side']} "
          f"({st['packed_share']:.1%} packed); wrote {a.out}")
    if a.level:
        lv = st["level"]
        print(f"levelled {lv['seam_pairs']} seam pairs over {lv['unknowns']} unknowns in "
              f"{lv['cg_iterations']} CG iterations: seam RMS {lv['seam_rms_before']:.3f} -> "
              f"{lv['seam_rms_after']:.3f}")


if __name__ == "__main__":
    main()
