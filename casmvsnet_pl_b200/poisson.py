"""Mesh any point cloud on the GPU: normal estimation and Poisson surface reconstruction on a
dense node grid (csrc/poisson.cu), extracted by the TSDF mesher's marching cubes (csrc/mesh.cu).
oracle/poisson_oracle.py restates every stage in numpy float64.

    verts, colours, faces, stats = poisson_mesh(xyz, rgb, normals=None, cam_centres=C, depth=9)
    mesh.write_mesh_ply("mesh.ply", verts, colours, faces)

    python -m casmvsnet_pl_b200.poisson --ply X.ply --out mesh.ply [--cams DIR] [--depth 9]

The rules (README, "Mesh any cloud"): E is the largest extent of the finite points' bounding box
and c its centre; h = float32(1.1 E / 2^depth); the grid is a cube of N = 2^depth nodes per axis,
node ijk at world ijk h, first node floor(c / h) - N/2 per axis.  Without normals, each point
takes the smallest-eigenvalue eigenvector of the covariance of the points in the 3x3x3 cells
around its cell (cell = round(p / h)), oriented toward the nearest camera centre; a point whose
block holds < 3 points or has covariance rank < 2 is dropped.  V = sum w n, W = sum w and
C = sum w rgb are splatted trilinearly, b = div V, and L chi = b (7-point Laplacian, chi = 0 on
the outer layer) is solved by V(2,2) multigrid cycles until ||r|| / ||b|| <= 1e-5 or 40 cycles.
f = chi - iso (iso = mean chi at the points) is meshed where the 5x5x5 box sum of W is positive.
With a point weight alpha > 0 (screened Poisson, README "Screening"), the unscreened chi0 gives the
target t = iso(chi0), and L chi - gamma S chi = b - gamma t Phi (S_ij = sum_p phi_i phi_j, Phi_i =
sum_p phi_i over the trilinear weights, gamma = alpha (n_s / n) / h^2, n_s the number of splat
cells) is solved from chi0 by 8-colour Gauss-Seidel V(2,2) cycles; its iso level is meshed."""
from __future__ import annotations

import argparse
import ctypes
import glob
import math
import os
import sys

import numpy as np
import torch

from . import _lib, io, mesh

MIN_DEPTH, MAX_DEPTH, DEFAULT_DEPTH = 6, 10, 9
TOL, MAX_CYCLES = 1e-5, 40
PRE_SWEEPS, POST_SWEEPS, COARSEST, COARSEST_SWEEPS = 2, 2, 8, 50
# peak device bytes per grid node (splat: cell map 4 + V 12 + W 4 + C 12 + b 4; the solve, with
# chi 8 + b 4 + three float fields 12 + coarse levels, stays below it) and per input point
# (keys and sort 24, sorted copies of the point, normal and colour 27, normals 12, cell maps 8)
BYTES_PER_NODE = 36
BYTES_PER_POINT = 72
# screening: per grid node the int32 cell map, u8 corner mask and int32 stencil row of every level
# (9 B x 8/7); per level-0 splat cell its 27 double moments with those of the coarser levels
# (216 B x 4/3), and its at most 8 surface nodes with their f32 stencils on every level
# (8 x 116 B x 4/3) and f64 stencils on level 0 (8 x 216 B)
SCREEN_BYTES_PER_NODE = 11
SCREEN_BYTES_PER_CELL = 3300
_KEY_NONE = torch.iinfo(torch.int64).max
_BIAS = 1 << 20


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bytes_needed(depth, n_points, n_bricks=0, screen=False, n_cells=0):
    """Device bytes of a call: the dense grid, the points, and the brick volume with its
    marching-cubes buffers (mesh.BYTES_PER_VOXEL per brick voxel); with `screen`, also the
    screening's cell maps and the moments of its n_cells splat cells (0 before they are known)."""
    per_node = BYTES_PER_NODE + (SCREEN_BYTES_PER_NODE if screen else 0)
    return (per_node * (1 << depth) ** 3 + BYTES_PER_POINT * n_points
            + mesh.BYTES_PER_VOXEL * 512 * n_bricks + SCREEN_BYTES_PER_CELL * n_cells)


def _check_point_weight(point_weight):
    if isinstance(point_weight, bool) or not isinstance(point_weight, (int, float, np.integer, np.floating)) \
            or not math.isfinite(point_weight) or point_weight < 0:
        raise ValueError(f"point_weight must be a finite number >= 0, got {point_weight!r}")


def _check_depth(depth):
    if not (isinstance(depth, (int, np.integer)) and MIN_DEPTH <= depth <= MAX_DEPTH):
        raise ValueError(f"depth must be an integer in {MIN_DEPTH}..{MAX_DEPTH}, got {depth!r}")


def grid(xyz, depth):
    """(n,3) float32 CUDA points -> dict(h, N, lo (3 ints), centre (3 floats)) of the finite
    points.  Raises ValueError when there is no finite point or the bounding box is flat in
    every direction (E = 0)."""
    _check_depth(depth)
    fin = torch.isfinite(xyz).all(1)
    p = xyz[fin]
    if p.numel() == 0:
        raise ValueError("the cloud has no finite point")
    mn = p.amin(0).double().cpu().numpy()
    mx = p.amax(0).double().cpu().numpy()
    E = float((mx - mn).max())
    if E == 0:
        raise ValueError("the cloud's bounding box has zero extent (all points coincide)")
    N = 1 << depth
    h = float(np.float32(1.1 * E / N))
    c = (mn + mx) / 2
    lo = [int(v) for v in np.floor(c / h).astype(np.int64) - N // 2]
    if min(lo) < -8 * _BIAS or max(lo) + N > 8 * (_BIAS - 1):
        raise ValueError(f"the cloud lies too far from the origin for its extent ({E:g}): its grid "
                         "nodes leave the mesh volume's index range")
    return dict(h=h, N=N, lo=lo, centre=[float(v) for v in c])


def _check_fits(depth, n_points, budget, n_bricks=0, screen=False, n_cells=0):
    """Refuse a call whose grid, points and bricks (0 before they are known), and with `screen`
    the screening buffers, need more than `budget` bytes, or whose bricks exceed mesh.MAX_BRICKS,
    naming the largest depth that fits.  Bricks and splat cells lie on the surface: at a lower
    depth their number is estimated as a quarter per level."""
    def bricks_at(d):
        return math.ceil(n_bricks / 4 ** (depth - d))

    def fits(d):
        return (bricks_at(d) <= mesh.MAX_BRICKS
                and _bytes_needed(d, n_points, bricks_at(d), screen,
                                  math.ceil(n_cells / 4 ** (depth - d))) <= budget)
    if fits(depth):
        return
    need = _bytes_needed(depth, n_points, n_bricks, screen, n_cells)
    lower = [d for d in range(MIN_DEPTH, depth) if fits(d)]
    hint = (f"depth {lower[-1]} would fit" if lower else
            f"no depth from {MIN_DEPTH} fits; thin the cloud")
    what = f"{n_points} points" + (f" and {n_bricks} bricks" if n_bricks else "")
    if screen:
        what += " with screening" + (f" of {n_cells} splat cells" if n_cells else "")
    if n_bricks > mesh.MAX_BRICKS:
        raise _lib.CasMVSError(f"the Poisson mesh at depth {depth} with {what} exceeds the mesh "
                               f"volume's {mesh.MAX_BRICKS} bricks; {hint}")
    raise _lib.CasMVSError(
        f"the Poisson grid at depth {depth} with {what} needs {need / 2**30:.2f} GiB but "
        f"{max(budget, 0) / 2**30:.2f} GiB are available; {hint}")


def _cells(keys):
    """Sorted keys -> (cell keys, counts, start offsets (n_cells + 1) int32)."""
    cells, counts = torch.unique_consecutive(keys, return_counts=True)
    start = torch.zeros(len(cells) + 1, dtype=torch.int32, device=keys.device)
    start[1:] = torch.cumsum(counts, 0)
    return cells, counts, start


def _cell_map(cells, N):
    cell_of = torch.full((N ** 3,), -1, dtype=torch.int32, device=cells.device)
    cell_of[cells] = torch.arange(len(cells), dtype=torch.int32, device=cells.device)
    return cell_of


def _vcycle(l, sizes, hs, e, rhs, tmp):
    """One V(2,2) cycle for L e[l] = rhs[l] from e[l] = 0 on level l (level 0 the finest)."""
    lib, st, n = _lib.load(), _stream(), sizes[l]
    if l == len(sizes) - 1:
        _lib.check(lib.casmvs_poisson_smooth(_ptr(e[l]), _ptr(rhs[l]), n, l, hs[l], COARSEST_SWEEPS,
                                             1, st), "poisson_smooth")
        return
    _lib.check(lib.casmvs_poisson_smooth(_ptr(e[l]), _ptr(rhs[l]), n, l, hs[l], PRE_SWEEPS, 1, st),
               "poisson_smooth")
    _lib.check(lib.casmvs_poisson_mg_residual(_ptr(e[l]), _ptr(rhs[l]), n, l, hs[l], _ptr(tmp[l]), st),
               "poisson_mg_residual")
    _lib.check(lib.casmvs_poisson_restrict(_ptr(tmp[l]), n, _ptr(rhs[l + 1]), st), "poisson_restrict")
    _vcycle(l + 1, sizes, hs, e, rhs, tmp)
    _lib.check(lib.casmvs_poisson_prolong_add(_ptr(e[l + 1]), sizes[l + 1], _ptr(e[l]), l, st),
               "poisson_prolong_add")
    _lib.check(lib.casmvs_poisson_smooth(_ptr(e[l]), _ptr(rhs[l]), n, l, hs[l], POST_SWEEPS, 0, st),
               "poisson_smooth")


def _solve(b, bb, N, h, ws):
    """V(2,2) multigrid for L chi = b -> (chi (N^3) float64, cycles, ||r|| / ||b|| before each
    cycle and at the end (cycles + 1 values)).  chi and the residual are kept in double on the
    finest level; each cycle solves for the correction in float32."""
    lib, st, dev = _lib.load(), _stream(), b.device
    sizes = [N >> l for l in range(0, 32) if (N >> l) >= COARSEST]
    f32 = dict(dtype=torch.float32, device=dev)
    chi = torch.zeros(N ** 3, dtype=torch.float64, device=dev)
    bn = math.sqrt(bb)
    if bn == 0:
        return chi, 0, [0.0]
    rhs = [torch.empty(n ** 3, **f32) for n in sizes]
    e = [torch.empty(n ** 3, **f32) for n in sizes]
    tmp = [torch.empty(n ** 3, **f32) for n in sizes[:-1]]
    hs = [float(np.float32(h * (1 << l))) for l in range(len(sizes))]
    rr = torch.zeros(1, dtype=torch.float64, device=dev)
    cycles = 0
    ratios = []
    while True:
        _lib.check(lib.casmvs_poisson_residual(_ptr(chi), _ptr(b), N, h, _ptr(rhs[0]), _ptr(ws),
                                               _ptr(rr), st), "poisson_residual")
        ratios.append(math.sqrt(float(rr.item())) / bn)
        if ratios[-1] <= TOL or cycles == MAX_CYCLES:
            return chi, cycles, ratios
        _vcycle(0, sizes, hs, e, rhs, tmp)
        _lib.check(lib.casmvs_poisson_accumulate(_ptr(chi), _ptr(e[0]), N, st), "poisson_accumulate")
        cycles += 1


def _corner_mask(cells, n):
    """u8 (n^3): bit d (d = 4 dx + 2 dy + dz) of node c + d set for every cell c; corners at index n
    (a coarse level's unstored Dirichlet node) are left out."""
    x, y, z = cells // (n * n), (cells // n) % n, cells % n
    mask = torch.zeros(n ** 3, dtype=torch.uint8, device=cells.device)
    for d in range(8):
        X, Y, Z = x + (d >> 2), y + ((d >> 1) & 1), z + (d & 1)
        idx = ((X * n + Y) * n + Z)[(X < n) & (Y < n) & (Z < n)]
        mask[idx] |= 1 << d                                   # each (node, d) once: no race
    return mask


def _stencils(cmap, mask, mom, n, double):
    """The S stencils of a level's surface nodes (mask != 0) -> (srow (n^3) int32, f32 stencils
    (s,27), f64 stencils (s,27) or None)."""
    lib, st, dev = _lib.load(), _stream(), mask.device
    nodes = torch.nonzero(mask).reshape(-1)                   # sorted
    srow = torch.full((n ** 3,), -1, dtype=torch.int32, device=dev)
    srow[nodes] = torch.arange(len(nodes), dtype=torch.int32, device=dev)
    s32 = torch.empty(len(nodes), 27, dtype=torch.float32, device=dev)
    s64 = torch.empty(len(nodes), 27, dtype=torch.float64, device=dev) if double else None
    _lib.check(lib.casmvs_poisson_screen_stencil(_ptr(nodes), len(nodes), _ptr(mask), _ptr(cmap),
                                                 _ptr(mom), n, _ptr(s32), _ptr(s64), st),
               "poisson_screen_stencil")
    return srow, s32, s64


def _screen_levels(p, N, h, lo, check=None):
    """Splat cells and their moments on every level -> ([dict(keys, map, mask, moments, srow,
    stencil (f32), stencil64 (level 0 only))] per level, level 0 first, down to COARSEST^3).
    check(n_cells), when given, runs once the cells are counted, before the levels are built."""
    lib, st, dev = _lib.load(), _stream(), p.device
    keys = torch.empty(len(p), dtype=torch.int64, device=dev)
    _lib.check(lib.casmvs_poisson_screen_keys(_ptr(p), len(p), h, *lo, N, _ptr(keys), st),
               "poisson_screen_keys")
    keys, order = torch.sort(keys, stable=True)
    n_ok = int((keys != _KEY_NONE).sum())
    keys, order = keys[:n_ok], order[:n_ok].to(torch.int32)
    cells, _, start = _cells(keys)
    del keys
    if check is not None:
        check(len(cells))
    mom = torch.empty(len(cells), 27, dtype=torch.float64, device=dev)
    _lib.check(lib.casmvs_poisson_screen_moments(_ptr(p), _ptr(order), _ptr(start), len(cells), h,
                                                 *lo, _ptr(mom), st), "poisson_screen_moments")
    del order, start
    levels = [(cells, _cell_map(cells, N), _corner_mask(cells, N), mom)]
    n = N
    while n // 2 >= COARSEST:
        ck, cmap, _, cmom = levels[-1]
        m = n // 2
        x, y, z = ck // (n * n), (ck // n) % n, ck % n
        pk = torch.unique((((x >> 1) * m + (y >> 1)) * m + (z >> 1)))        # sorted
        pm = torch.empty(len(pk), 27, dtype=torch.float64, device=dev)
        _lib.check(lib.casmvs_poisson_screen_coarsen(_ptr(cmap), _ptr(cmom), n, _ptr(pk), len(pk),
                                                     _ptr(pm), st), "poisson_screen_coarsen")
        levels.append((pk, _cell_map(pk, m), _corner_mask(pk, m), pm))
        n = m
    out = []
    for l, (k, cmap, mask, mom) in enumerate(levels):
        srow, s32, s64 = _stencils(cmap, mask, mom, N >> l, l == 0)
        out.append(dict(keys=k, map=cmap, mask=mask, moments=mom, srow=srow, stencil=s32,
                        stencil64=s64))
    return out


def _screen_vcycle(l, sizes, hs, g, levels, e, rhs, tmp):
    """One screened V(2,2) cycle for (L_l - gamma_l S_l) e[l] = rhs[l] from e[l] = 0."""
    lib, st, n = _lib.load(), _stream(), sizes[l]
    lv = levels[l]
    ops = (_ptr(lv["mask"]), _ptr(lv["srow"]), _ptr(lv["stencil"]), n, l, hs[l], g)
    if l == len(sizes) - 1:
        _lib.check(lib.casmvs_poisson_screen_smooth(_ptr(e[l]), _ptr(rhs[l]), *ops, COARSEST_SWEEPS,
                                                    1, st), "poisson_screen_smooth")
        return
    _lib.check(lib.casmvs_poisson_screen_smooth(_ptr(e[l]), _ptr(rhs[l]), *ops, PRE_SWEEPS, 1, st),
               "poisson_screen_smooth")
    _lib.check(lib.casmvs_poisson_screen_mg_residual(_ptr(e[l]), _ptr(rhs[l]), *ops, _ptr(tmp[l]), st),
               "poisson_screen_mg_residual")
    _lib.check(lib.casmvs_poisson_restrict(_ptr(tmp[l]), n, _ptr(rhs[l + 1]), st), "poisson_restrict")
    _screen_vcycle(l + 1, sizes, hs, g, levels, e, rhs, tmp)
    _lib.check(lib.casmvs_poisson_prolong_add(_ptr(e[l + 1]), sizes[l + 1], _ptr(e[l]), l, st),
               "poisson_prolong_add")
    _lib.check(lib.casmvs_poisson_screen_smooth(_ptr(e[l]), _ptr(rhs[l]), *ops, POST_SWEEPS, 0, st),
               "poisson_screen_smooth")


def _screen_solve(chi, b_s, bb, N, h, g, levels, ws):
    """Screened V(2,2) multigrid from chi (updated in place) -> (cycles, ratios), as _solve."""
    lib, st, dev = _lib.load(), _stream(), b_s.device
    sizes = [N >> l for l in range(len(levels))]
    f32 = dict(dtype=torch.float32, device=dev)
    bn = math.sqrt(bb)
    if bn == 0:
        return 0, [0.0]
    rhs = [torch.empty(n ** 3, **f32) for n in sizes]
    e = [torch.empty(n ** 3, **f32) for n in sizes]
    tmp = [torch.empty(n ** 3, **f32) for n in sizes[:-1]]
    hs = [float(np.float32(h * (1 << l))) for l in range(len(sizes))]
    rr = torch.zeros(1, dtype=torch.float64, device=dev)
    lv = levels[0]
    cycles, ratios = 0, []
    while True:
        _lib.check(lib.casmvs_poisson_screen_residual(_ptr(chi), _ptr(b_s), _ptr(lv["mask"]),
                                                      _ptr(lv["srow"]), _ptr(lv["stencil64"]), N, h,
                                                      g, _ptr(rhs[0]), _ptr(ws), _ptr(rr), st),
                   "poisson_screen_residual")
        ratios.append(math.sqrt(float(rr.item())) / bn)
        if ratios[-1] <= TOL or cycles == MAX_CYCLES:
            return cycles, ratios
        _screen_vcycle(0, sizes, hs, g, levels, e, rhs, tmp)
        _lib.check(lib.casmvs_poisson_accumulate(_ptr(chi), _ptr(e[0]), N, st), "poisson_accumulate")
        cycles += 1


def poisson_mesh(xyz, rgb=None, normals=None, cam_centres=None, depth=DEFAULT_DEPTH, max_bytes=None,
                 log=print, fields=None, events=None, point_weight=0.0):
    """Poisson surface of the points xyz (n,3) float32 CUDA tensor, with colours rgb (n,3) uint8
    (None: white) and either normals (n,3) float32 (normalised; zero-length ones are dropped) or
    the camera centres cam_centres (k,3) that estimated normals are oriented toward.
    -> (verts (V,3) float32, colours (V,3) uint8, faces (F,3) int32 on the device, stats dict:
    h, N, depth, points, dropped, cycles, residual, ratios (||r|| / ||b|| before each cycle and
    at the end), iso, bricks, vertices, triangles).
    Raises ValueError for a depth outside 6..10, a cloud without a finite point or with zero
    extent, or neither normals nor cameras; CasMVSError when the grid, or once they are known the
    grid and the mesh bricks, would not fit in free device memory (or `max_bytes`), naming the
    largest depth that would.  A solve that stops at 40 cycles
    above the tolerance is logged, not refused.  `fields`, a dict, receives the intermediate
    device tensors (index and normals of the kept points in sorted order, V, W, C, b, chi, iso,
    keep, and the brick volume keys, tsdf, weight, color) for checking the stages; `events`, a list, receives (phase, CUDA event) pairs recorded
    at the start and at the end of each phase, for timing.
    point_weight (alpha, finite, >= 0; ValueError otherwise) > 0 screens the solve: stats gain
    point_weight, target (t, the unscreened iso level), screened_cycles and screened_ratios
    (cycles and ratios stay the unscreened solve's; iso is the screened field's), fields gain
    chi0 (unscreened), b_s, g (alpha n_s / n) and levels ([(cell keys, moments)] per level),
    events a "screen" phase after "solve".  alpha = 0 runs the unscreened code alone."""
    _check_depth(depth)
    _check_point_weight(point_weight)
    screen = point_weight > 0
    xyz = mesh._check_cuda("xyz", xyz, torch.float32, (3,)).reshape(-1, 3)
    dev = xyz.device
    if normals is None and cam_centres is None:
        raise ValueError("poisson_mesh needs normals or camera centres to orient estimated normals")
    if normals is not None:
        normals = mesh._check_cuda("normals", normals, torch.float32, (3,)).reshape(-1, 3)
        if len(normals) != len(xyz):
            raise ValueError("normals must have one row per point")
    if rgb is not None:
        rgb = mesh._check_cuda("rgb", rgb, torch.uint8, (3,)).reshape(-1, 3)
        if len(rgb) != len(xyz):
            raise ValueError("rgb must have one row per point")
    lib = _lib.load()

    def mark(phase):
        if events is not None:
            events.append((phase, torch.cuda.Event(enable_timing=True)))
            events[-1][1].record()
    with torch.cuda.device(dev):
        mark("start")
        g = grid(xyz, depth)
        h, N, lo = g["h"], g["N"], g["lo"]
        n_in = len(xyz)
        budget = mesh.device_budget(dev, max_bytes)
        _check_fits(depth, n_in, budget, screen=screen)
        st = _stream()
        # cells: sort the points by cell key, stably; dropped points sort last
        keys = torch.empty(n_in, dtype=torch.int64, device=dev)
        unit = torch.empty(n_in, 3, dtype=torch.float32, device=dev) if normals is not None else None
        _lib.check(lib.casmvs_poisson_cell_keys(_ptr(xyz), _ptr(normals), n_in, h, *lo, N, _ptr(keys),
                                                _ptr(unit), st), "poisson_cell_keys")
        keys, perm = torch.sort(keys, stable=True)
        n_ok = int((keys != _KEY_NONE).sum())
        keys, perm = keys[:n_ok], perm[:n_ok]
        p = xyz[perm]
        col = rgb[perm] if rgb is not None else None
        nrm = unit[perm] if unit is not None else None
        del unit
        cells, counts, start = _cells(keys)
        mark("sort")
        if nrm is None and n_ok:
            cams = torch.as_tensor(np.asarray(cam_centres, np.float64).reshape(-1, 3), device=dev)
            if len(cams) == 0:
                raise ValueError("cam_centres is empty")
            cell_of = _cell_map(cells, N)
            mom = torch.empty(len(cells), 10, dtype=torch.float64, device=dev)
            _lib.check(lib.casmvs_poisson_cell_moments(_ptr(p), _ptr(start), len(cells), *g["centre"],
                                                       _ptr(mom), st), "poisson_cell_moments")
            mark("moments")
            cn = torch.empty(len(cells), 3, dtype=torch.float64, device=dev)
            cok = torch.empty(len(cells), dtype=torch.uint8, device=dev)
            _lib.check(lib.casmvs_poisson_cell_normals(_ptr(cells), _ptr(cell_of), _ptr(mom),
                                                       len(cells), N, _ptr(cn), _ptr(cok), st),
                       "poisson_cell_normals")
            del cell_of, mom
            pcell = torch.repeat_interleave(torch.arange(len(cells), dtype=torch.int32, device=dev),
                                            counts)
            nrm = torch.empty(n_ok, 3, dtype=torch.float32, device=dev)
            _lib.check(lib.casmvs_poisson_orient(_ptr(p), _ptr(pcell), _ptr(cn), n_ok, _ptr(cams),
                                                 len(cams), _ptr(nrm), st), "poisson_orient")
            keep = cok.bool()[pcell]
            del pcell, cn
            if not bool(keep.all()):
                p, nrm, keys, perm = p[keep], nrm[keep], keys[keep], perm[keep]
                col = col[keep] if col is not None else None
                cells, counts, start = _cells(keys)
        mark("normals")
        n_kept = len(p)
        dropped = n_in - n_kept
        if n_kept == 0:
            raise ValueError("no point of the cloud has a usable normal")
        if fields is not None:
            fields.update(index=perm, normals=nrm)
        del perm
        # splat and divergence
        f32 = dict(dtype=torch.float32, device=dev)
        cell_of = _cell_map(cells, N)
        V, W, C = torch.empty(N ** 3, 3, **f32), torch.empty(N ** 3, **f32), torch.empty(N ** 3, 3, **f32)
        _lib.check(lib.casmvs_poisson_splat(_ptr(p), _ptr(nrm), _ptr(col), _ptr(start), _ptr(cell_of),
                                            N, h, *lo, _ptr(V), _ptr(W), _ptr(C), st), "poisson_splat")
        del cell_of, keys, cells, counts, start, nrm, col
        mark("splat")
        ws = torch.empty(lib.casmvs_poisson_workspace_bytes(N ** 3) // 8, dtype=torch.float64,
                         device=dev)
        bb = torch.zeros(1, dtype=torch.float64, device=dev)
        b = torch.empty(N ** 3, **f32)
        _lib.check(lib.casmvs_poisson_rhs(_ptr(V), N, h, _ptr(b), _ptr(ws), _ptr(bb), st), "poisson_rhs")
        if fields is not None:
            fields.update(V=V, W=W, C=C, b=b)
        del V
        mark("rhs")
        # trim, bricks and colour, before the solve so that W and C are freed for it
        keepn = torch.empty(N ** 3, dtype=torch.uint8, device=dev)
        work = torch.empty(N ** 3, dtype=torch.uint8, device=dev)
        _lib.check(lib.casmvs_poisson_trim(_ptr(W), N, _ptr(keepn), _ptr(work), st), "poisson_trim")
        del work
        b0 = [v // 8 for v in lo]
        nbk = [(v + N - 1) // 8 - v // 8 + 1 for v in lo]
        flags = torch.empty(nbk[0], nbk[1], nbk[2], dtype=torch.uint8, device=dev)
        _lib.check(lib.casmvs_poisson_brick_flags(_ptr(keepn), N, *lo, *b0, *nbk, _ptr(flags), st),
                   "poisson_brick_flags")
        bi = torch.nonzero(flags).to(torch.int64) + torch.tensor(b0, device=dev) + _BIAS   # sorted
        bkeys = ((bi[:, 0] << 42) | (bi[:, 1] << 21) | bi[:, 2]).contiguous()
        del flags, bi
        nb = len(bkeys)
        _check_fits(depth, n_in, budget, nb, screen=screen)
        nbr = torch.empty(nb, 7, dtype=torch.int32, device=dev)
        _lib.check(lib.casmvs_mesh_brick_neighbors(_ptr(bkeys), nb, _ptr(nbr), st),
                   "mesh_brick_neighbors")
        tsdf, weight = torch.empty(nb * 512, **f32), torch.empty(nb * 512, **f32)
        color = torch.empty(nb * 512, 3, **f32)
        _lib.check(lib.casmvs_poisson_fill_bricks(_ptr(bkeys), nb, _ptr(keepn), _ptr(W), _ptr(C), N,
                                                  *lo, _ptr(weight), _ptr(color), st),
                   "poisson_fill_bricks")
        if fields is not None:
            fields.update(keep=keepn)
        del keepn, W, C
        mark("trim_bricks")
        # solve, iso level, field
        chi, cycles, ratios = _solve(b, float(bb.item()), N, h, ws)
        ratio = ratios[-1]
        if not screen:
            del b, ws
        ws_p = torch.empty(max(1, lib.casmvs_poisson_workspace_bytes(n_kept) // 8),
                           dtype=torch.float64, device=dev)
        s = torch.zeros(1, dtype=torch.float64, device=dev)
        _lib.check(lib.casmvs_poisson_iso_sum(_ptr(chi), _ptr(p), n_kept, N, h, *lo, _ptr(ws_p), _ptr(s),
                                              st), "poisson_iso_sum")
        iso = float(s.item()) / n_kept
        target, s_cycles, s_ratios = None, 0, []
        if screen:
            # screening: the target t = iso(chi0), then L chi - gamma S chi = b - gamma t Phi from chi0
            mark("solve")
            target = iso
            levels = _screen_levels(p, N, h, lo, check=lambda c: _check_fits(
                depth, n_in, budget, nb, screen=True, n_cells=c))
            n_s = len(levels[0]["keys"])
            g = point_weight * n_s / n_kept
            if fields is not None:
                fields.update(chi0=chi.clone(), g=g,
                              levels=[(lv["keys"], lv["moments"]) for lv in levels])
            b_s = torch.empty(N ** 3, **f32)
            lv = levels[0]
            _lib.check(lib.casmvs_poisson_screen_rhs(_ptr(b), _ptr(lv["mask"]), _ptr(lv["map"]),
                                                     _ptr(lv["moments"]), N, g / (h * h) * target,
                                                     _ptr(b_s), _ptr(ws), _ptr(bb), st),
                       "poisson_screen_rhs")
            del b
            for lv in levels:                                  # the solve reads the stencils
                lv["map"] = None
            if fields is not None:
                fields.update(b_s=b_s, bb_s=float(bb.item()))
            s_cycles, s_ratios = _screen_solve(chi, b_s, float(bb.item()), N, h, g, levels, ws)
            del b_s, ws, levels, lv
            _lib.check(lib.casmvs_poisson_iso_sum(_ptr(chi), _ptr(p), n_kept, N, h, *lo, _ptr(ws_p),
                                                  _ptr(s), st), "poisson_iso_sum")
            iso = float(s.item()) / n_kept
        if fields is not None:
            fields.update(chi=chi, iso=iso)
        _lib.check(lib.casmvs_poisson_fill_tsdf(_ptr(bkeys), nb, _ptr(weight), _ptr(chi), iso, N, *lo,
                                                _ptr(tsdf), st), "poisson_fill_tsdf")
        if fields is not None:
            fields.update(keys=bkeys, tsdf=tsdf, weight=weight, color=color)
        del chi, p, ws_p
        mark("screen" if screen else "solve")
        verts, colours, faces = mesh.extract_bricks(bkeys, nbr, h, tsdf, weight, color)
        mark("extract")
    if ratio > TOL and log is not None:
        log(f"poisson: the multigrid solve stopped after {cycles} cycles at residual ratio "
            f"{ratio:.3g} (> {TOL:g}); the mesh is from the unconverged field")
    if screen and s_ratios[-1] > TOL and log is not None:
        log(f"poisson: the screened solve stopped after {s_cycles} cycles at residual ratio "
            f"{s_ratios[-1]:.3g} (> {TOL:g}); the mesh is from the unconverged field")
    stats = dict(h=h, N=N, depth=depth, points=n_kept, dropped=dropped, cycles=cycles,
                 residual=ratio, ratios=ratios, iso=iso, bricks=nb, vertices=len(verts),
                 triangles=len(faces), point_weight=float(point_weight), target=target,
                 screened_cycles=s_cycles, screened_ratios=s_ratios)
    return verts, colours, faces, stats


# ------------------------------------------------------------------------------ command line
def read_cloud(path):
    """A point PLY -> (xyz (n,3) float32, rgb (n,3) uint8 or None, normals (n,3) float32 or None)
    as numpy arrays."""
    v = io.read_ply(path)
    names = v.dtype.names or ()
    if not all(a in names for a in ("x", "y", "z")):
        raise ValueError(f"{path}: the vertex element has no x, y, z")

    def cols(*a):
        return np.stack([v[k] for k in a], axis=1) if all(k in names for k in a) else None
    xyz = cols("x", "y", "z").astype(np.float32)
    rgb = cols("red", "green", "blue")
    nrm = cols("nx", "ny", "nz")
    return (xyz, None if rgb is None else rgb.astype(np.uint8),
            None if nrm is None else nrm.astype(np.float32))


def camera_centres(cam_dir):
    """Centres -R^T t of the MVSNet *_cam.txt files in cam_dir (sorted by name) -> (k,3) float64."""
    files = sorted(glob.glob(os.path.join(cam_dir, "*_cam.txt")))
    if not files:
        raise ValueError(f"{cam_dir}: no *_cam.txt camera files")
    out = []
    for f in files:
        _, E, _ = io.read_cam_file(f)
        E = E.astype(np.float64)
        out.append(-E[:3, :3].T @ E[:3, 3])
    return np.stack(out)


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Mesh a point cloud by Poisson surface reconstruction "
                                             "on the GPU.")
    ap.add_argument("--ply", required=True, help="the point cloud (PLY, with or without normals)")
    ap.add_argument("--out", required=True, help="the mesh PLY to write")
    ap.add_argument("--cams", default=None,
                    help="a directory of MVSNet *_cam.txt files: the cameras that orient estimated "
                         "normals (needed when the PLY has no nx, ny, nz)")
    ap.add_argument("--depth", type=int, default=DEFAULT_DEPTH,
                    help=f"grid depth: 2^depth nodes per axis, {MIN_DEPTH}..{MAX_DEPTH}")
    ap.add_argument("--point_weight", type=float, default=0.0,
                    help="screening weight alpha >= 0: pulls the surface through the samples "
                         "(0, the default: unscreened Poisson)")
    a = ap.parse_args(argv)
    if not MIN_DEPTH <= a.depth <= MAX_DEPTH:
        ap.error(f"--depth must be in {MIN_DEPTH}..{MAX_DEPTH}")
    if not (math.isfinite(a.point_weight) and a.point_weight >= 0):
        ap.error("--point_weight must be a finite number >= 0")
    return a, ap


def main(argv=None):
    a, ap = parse_args(argv)
    xyz, rgb, nrm = read_cloud(a.ply)
    if nrm is None and a.cams is None:
        ap.error(f"{a.ply} has no normals (nx, ny, nz): give --cams DIR, the camera files that "
                 "orient the estimated normals")
    cams = camera_centres(a.cams) if nrm is None else None
    dev = "cuda"

    def cuda(x):
        return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    verts, colours, faces, st = poisson_mesh(cuda(xyz), cuda(rgb), cuda(nrm), cams, a.depth,
                                             point_weight=a.point_weight)
    d = os.path.dirname(os.path.abspath(a.out))
    os.makedirs(d, exist_ok=True)
    mesh.write_mesh_ply(a.out, verts, colours, faces)
    print(f"{a.out}: depth {st['depth']} (h {st['h']:.6g}, {st['N']}^3 nodes), {st['points']} points "
          f"({st['dropped']} dropped), {st['cycles']} multigrid cycles (residual ratio "
          f"{st['residual']:.3g}), {st['bricks']} bricks, {st['vertices']} vertices, "
          f"{st['triangles']} triangles" + (f", screened (point weight {a.point_weight:g}) in "
                                            f"{st['screened_cycles']} cycles"
                                            if a.point_weight > 0 else ""))


if __name__ == "__main__":
    sys.exit(main())
