"""Poisson reconstruction per element against float64 (oracle/poisson_fp64.py) on the GPU:

* every multigrid kernel through the C ABI at depths 6-10 and at every level, on a real
  right-hand side (a splatted sphere) and seeded random fields: smooth (one sweep, both zero_first
  paths, so the one-block coarsest kernel at n = 8), mg_residual, restrict, prolong_add, residual
  and ||r||^2, rhs and ||b||^2, accumulate, splat, trim and the iso sum.  Depths 6-8 on the full
  grid, 9 and 10 in windows (corners, face centres, the surface and the last x-slabs, where a
  depth-10 V offset passes 2^31 floats);
* the whole pipeline with ``fields=`` on a table of clouds, each named for its edge, at depths 7
  and 8 on the full grid, and at depth 9 in windows: every stage, the cycle count and each cycle's
  contraction against the float64 multigrid of the kernel's own b;
* depth 10 end to end without fields, with its wall time and peak device memory.

A summary table of the worst eps needed per kernel and depth is printed at the end."""
import collections
import time

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, mesh, poisson
from oracle import mesh_oracle as M
from oracle import poisson_fp64 as F
from oracle import poisson_oracle as O

DEV = "cuda:0"
TABLE = collections.defaultdict(dict)        # kernel -> depth -> worst eps needed


def _record(depth, *reps):
    for rep in reps:
        d = TABLE[rep.kernel]
        d[depth] = max(d.get(depth, 0.0), rep.eps_needed)
        assert rep.ok, f"depth {depth}: {rep.describe()}"


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if not TABLE:
        return
    depths = sorted({d for v in TABLE.values() for d in v})
    print("\n[poisson-fp64] worst eps needed per kernel and depth (eps in the last column)")
    print("| kernel | " + " | ".join(f"depth {d}" for d in depths) + " | eps |")
    print("|---|" + "---|" * (len(depths) + 1))
    for k in sorted(TABLE):
        row = [f"{TABLE[k][d]:.2e}" if d in TABLE[k] else "" for d in depths]
        print(f"| {k} | " + " | ".join(row) + f" | {F.EPS.get(k, F.EPS['reduction']):.2e} |")


def _ptr(t):
    return poisson._ptr(t)


def _st():
    return poisson._stream()


def _cuda(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


# ------------------------------------------------------------------------------- case table
def _offset_sphere(depth, shift, n=20_000, seed=0):
    p, nrm = O.sphere(n, seed=seed, noise=0.002)
    return (p.astype(np.float64) + shift).astype(np.float32), nrm


def cloud(name):
    """-> dict(xyz, rgb | None, normals | None, cams | None) of the named case."""
    rng = np.random.default_rng(11)
    if name == "lo_mixed":
        p, n = _offset_sphere(7, np.array([-3.0, 3.0, 0.37]))
        return dict(xyz=p, rgb=rng.integers(0, 256, (len(p), 3)).astype(np.uint8), normals=n, cams=None)
    if name == "dense_2m":
        # two far anchors stretch the grid 4x: hundreds of sphere points per cell
        p, n = O.sphere(2_000_000, seed=1, noise=0.001)
        p = np.concatenate([p, [[-4, -4, -4], [4, 4, 4]]]).astype(np.float32)
        n = np.concatenate([n, [[1, 0, 0], [1, 0, 0]]]).astype(np.float32)
        return dict(xyz=p, rgb=None, normals=n, cams=None)
    if name == "ties":
        p, n, _ = F.tie_cloud(7)
        return dict(xyz=p, rgb=None, normals=n, cams=None)
    if name in ("far_2p22", "far_guard"):
        target = 2.0 ** 22 if name == "far_2p22" else 8.3e6
        p, n = O.sphere(20_000, seed=2, noise=0.002)
        h = float(np.float32(1.1 * 2 / 128))
        p = (p.astype(np.float64) + target * h).astype(np.float32)
        return dict(xyz=p, rgb=None, normals=n, cams=None)
    if name == "blocks":
        sph, _ = O.sphere(30_000, seed=3, noise=0.001)
        line = np.stack([np.linspace(1.2, 1.3, 40), np.full(40, 1.25), np.full(40, 1.25)], 1)
        three = np.array([[-1.25, 1.25, -1.25], [-1.26, 1.25, -1.24], [-1.25, 1.26, -1.25]])
        dup = np.repeat(sph[:200], 3, axis=0)
        xs = rng.uniform(-0.5, 0.5, (4000, 2))
        plane = np.concatenate([xs + [0.0, -1.6], np.zeros((4000, 1))], 1)
        p = np.concatenate([sph, line, three, dup, plane]).astype(np.float32)
        cams = np.array([[0.0, -1.6, 3.0], [0.0, -1.6, -3.0], [6.0, 0.0, 0.0], [-6.0, 0.0, 0.0]])
        return dict(xyz=p, rgb=None, normals=None, cams=cams, line=line.astype(np.float32),
                    three=three.astype(np.float32))
    if name == "bad_values":
        p, n = O.sphere(20_000, seed=4, noise=0.002)
        p, n = p.copy(), n.copy()
        p[:10, 0] = np.nan
        p[10:20, 1] = np.inf
        p[20:30, 2] = -np.inf
        n[100:150] = 0
        n[150:200, 1] = np.nan
        return dict(xyz=p, rgb=None, normals=n, cams=None)
    if name == "rgb_extremes":
        p, n = O.sphere(20_000, seed=5, noise=0.002)
        rgb = np.where(rng.random((len(p), 1)) < 0.5, 0, 255).astype(np.uint8).repeat(3, 1)
        return dict(xyz=p, rgb=rgb, normals=n, cams=None)
    raise KeyError(name)


CASES = {
    "lo_mixed": dict(depths=(7, 8), edges=("lo_neg_not_mod8", "lo_pos_not_mod8")),
    "dense_2m": dict(depths=(7,), edges=("hundreds_per_cell",)),
    "ties": dict(depths=(7, 8), edges=("exact_ties", "exact_integers")),
    "far_2p22": dict(depths=(7,), edges=("quotient_2p22",)),
    "far_guard": dict(depths=(7,), edges=("quotient_near_guard",)),
    "blocks": dict(depths=(7, 8), edges=("collinear_block", "three_point_block", "duplicates",
                                         "planar_z0", "equidistant_cams")),
    "bad_values": dict(depths=(7, 8), edges=("nan_inf_points", "zero_nan_normals", "rgb_none")),
    "rgb_extremes": dict(depths=(7,), edges=("rgb_0_255",)),
}


def _q(c, depth):
    g = O.grid(c["xyz"], depth)
    p = c["xyz"][np.isfinite(c["xyz"]).all(1)]
    return p.astype(np.float64) / g["h"], g


def _isolated(c, group, depth):
    """No other point lies within 4 h (per axis) of the group, so the 3x3x3-cell blocks of its
    cells hold the group alone."""
    h = O.grid(c["xyz"], depth)["h"]
    p = c["xyz"][np.isfinite(c["xyz"]).all(1)].astype(np.float64)
    g = group.astype(np.float64)
    near = (np.abs(p[:, None, :] - g[None]) <= 4 * h).all(2).any(1)
    return near.sum() == len(g)


EDGES = {
    "lo_neg_not_mod8": lambda c, d: any(v < 0 and v % 8 for v in O.grid(c["xyz"], d)["lo"]),
    "lo_pos_not_mod8": lambda c, d: any(v > 0 and v % 8 for v in O.grid(c["xyz"], d)["lo"]),
    "hundreds_per_cell": lambda c, d: np.unique(O.flat(O.cell_index(c["xyz"], O.grid(c["xyz"], d)),
                                                       1 << d), return_counts=True)[1].max() >= 200,
    "exact_ties": lambda c, d: ((_q(c, d)[0] % 1 == 0.5) & (_q(c, d)[0].astype(np.float32) == _q(c, d)[0])).any(),
    "exact_integers": lambda c, d: ((_q(c, d)[0] % 1 == 0) & (np.abs(_q(c, d)[0]) > 0)).all(1).any(),
    "quotient_2p22": lambda c, d: 0.9 * 2 ** 22 <= np.abs(_q(c, d)[0]).max() <= 1.1 * 2 ** 22,
    "quotient_near_guard": lambda c, d: 8.0e6 <= np.abs(_q(c, d)[0]).max() < 2 ** 23,
    "collinear_block": lambda c, d: (c["normals"] is None and (np.ptp(c["line"][:, 1:], 0) == 0).all()
                                     and _isolated(c, c["line"], d)),
    "three_point_block": lambda c, d: c["normals"] is None and _isolated(c, c["three"], d),
    "duplicates": lambda c, d: len(np.unique(c["xyz"], axis=0)) < len(c["xyz"]),
    "planar_z0": lambda c, d: (c["xyz"][:, 2] == 0).sum() >= 4000,
    "equidistant_cams": lambda c, d: c["cams"] is not None and np.array_equal(
        c["cams"][0] * [1, 1, -1], c["cams"][1]),
    "nan_inf_points": lambda c, d: np.isnan(c["xyz"]).any() and np.isinf(c["xyz"]).any(),
    "zero_nan_normals": lambda c, d: (c["normals"] is not None and (c["normals"] == 0).all(1).any()
                                      and np.isnan(c["normals"]).any()),
    "rgb_none": lambda c, d: c["rgb"] is None,
    "rgb_0_255": lambda c, d: c["rgb"] is not None and {0, 255} <= set(np.unique(c["rgb"])),
}


def test_case_table_edges():
    """Every edge a case names holds by construction (checked at its first depth)."""
    for name, spec in CASES.items():
        c = cloud(name)
        for e in spec["edges"]:
            assert EDGES[e](c, spec["depths"][0]), f"{name}: edge {e} does not hold"
    assert {d for s in CASES.values() for d in s["depths"]} == {7, 8}


# ------------------------------------------------------------------------------- stage helpers
def _keys(xyz, nrm, g):
    lib = _lib.load()
    n = len(xyz)
    keys = torch.empty(n, dtype=torch.int64, device=DEV)
    unit = torch.empty(n, 3, dtype=torch.float32, device=DEV) if nrm is not None else None
    _lib.check(lib.casmvs_poisson_cell_keys(_ptr(xyz), _ptr(nrm), n, g["h"], *g["lo"], g["N"],
                                            _ptr(keys), _ptr(unit), _st()), "cell_keys")
    return keys, unit


def _splat(p, nrm, col, keys, g):
    lib = _lib.load()
    N = g["N"]
    cells, _, start = poisson._cells(keys)
    cell_of = poisson._cell_map(cells, N)
    f32 = dict(dtype=torch.float32, device=DEV)
    V, W, C = torch.empty(N ** 3, 3, **f32), torch.empty(N ** 3, **f32), torch.empty(N ** 3, 3, **f32)
    _lib.check(lib.casmvs_poisson_splat(_ptr(p), _ptr(nrm), _ptr(col), _ptr(start), _ptr(cell_of), N,
                                        g["h"], *g["lo"], _ptr(V), _ptr(W), _ptr(C), _st()), "splat")
    return V, W, C


def _wins(n, depth, surf=()):
    return None if depth <= 8 else F.windows(n, 32, surf)


def _surface_nodes(p, g, k=4):
    q = np.floor(p[:: max(1, len(p) // k)][:k].astype(np.float64) / g["h"]).astype(np.int64) - g["lo"]
    return [tuple(int(v) for v in r) for r in q]


# ------------------------------------------------------------------------------- per kernel, per level
def _level_kernels(depth, timing):
    lib, st = _lib.load(), _st()
    N = 1 << depth
    p, nrm = O.sphere(200_000, seed=depth, noise=0.002)
    g = O.grid(p, depth)
    g = dict(h=g["h"], N=N, lo=[int(v) for v in g["lo"]], centre=g["centre"])
    h = g["h"]
    surf = _surface_nodes(p, g)
    pd, nd = _cuda(p), _cuda(nrm)
    keys, unit = _keys(pd, nd, g)
    r1, r2 = F.check_cell_keys(pd, nd, h, g["lo"], N, keys, unit)
    _record(depth, r1, r2)
    keys, perm = torch.sort(keys, stable=True)
    ok = keys != F.KEY_NONE
    keys, perm = keys[ok], perm[ok]
    ps, ns = pd[perm].contiguous(), unit[perm].contiguous()
    V, W, C = _splat(ps, ns, None, keys, g)
    wins = _wins(N, depth, surf)
    reps = F.check_splat(ps, ns, None, h, g["lo"], N, V.view(N, N, N, 3), W.view(N, N, N),
                         C.view(N, N, N, 3), wins)
    _record(depth, *reps.values())
    keep = torch.empty(N ** 3, dtype=torch.uint8, device=DEV)
    work = torch.empty_like(keep)
    _lib.check(lib.casmvs_poisson_trim(_ptr(W), N, _ptr(keep), _ptr(work), st), "trim")
    del work
    _record(depth, F.check_trim(W.view(N, N, N), keep.view(N, N, N), N, wins))
    del keep, W, C
    ws = torch.empty(lib.casmvs_poisson_workspace_bytes(N ** 3) // 8, dtype=torch.float64, device=DEV)
    bb = torch.zeros(1, dtype=torch.float64, device=DEV)
    b = torch.empty(N ** 3, dtype=torch.float32, device=DEV)
    _lib.check(lib.casmvs_poisson_rhs(_ptr(V), N, h, _ptr(b), _ptr(ws), _ptr(bb), st), "rhs")
    _record(depth, F.check_rhs(V.view(N, N, N, 3), b.view(N, N, N), N, h, wins),
            F.check_reduction(float(bb), b.double() ** 2))
    del V
    gen = torch.Generator(device=DEV).manual_seed(depth)

    def rand(n, scale=1.0, dtype=torch.float32):
        return (torch.randn(n ** 3, generator=gen, device=DEV, dtype=torch.float32) * scale).to(dtype)
    bscale = float(b.abs().max())
    chi = rand(N, 1e-3 * bscale * h * h, torch.float64)
    r = torch.empty_like(b)
    rr = torch.zeros(1, dtype=torch.float64, device=DEV)
    _lib.check(lib.casmvs_poisson_residual(_ptr(chi), _ptr(b), N, h, _ptr(r), _ptr(ws), _ptr(rr), st),
               "residual")
    rep, _ = F.check_residual(chi.view(N, N, N), b.view(N, N, N), r.view(N, N, N), N, h, wins)
    r2 = r.double() ** 2
    _record(depth, rep, F.check_reduction(float(rr), r2, extra=2.0001 * F.U * float(r2.sum())))
    del r2, ws
    e = rand(N, 1e-3 * bscale * h * h)
    chi1 = chi.clone()
    _lib.check(lib.casmvs_poisson_accumulate(_ptr(chi1), _ptr(e), N, st), "accumulate")
    _record(depth, F.check_accumulate(chi.view(N, N, N), e.view(N, N, N), chi1.view(N, N, N), N, wins))
    del chi1, e
    # iso sum of the points against chi
    ws_p = torch.empty(max(1, lib.casmvs_poisson_workspace_bytes(len(ps)) // 8), dtype=torch.float64,
                       device=DEV)
    s = torch.zeros(1, dtype=torch.float64, device=DEV)
    _lib.check(lib.casmvs_poisson_iso_sum(_ptr(chi), _ptr(ps), len(ps), N, h, *g["lo"], _ptr(ws_p),
                                          _ptr(s), st), "iso_sum")
    _record(depth, *F.check_iso(chi, ps, h, g["lo"], N, float(s)))
    del chi, ws_p
    # every level: smooth (both paths), mg_residual, restrict, prolong_add
    hs = F.hs_levels(h, N)
    sizes = [N >> l for l in range(len(hs))]
    rhs = r
    del b
    for l, n in enumerate(sizes):
        wl = _wins(n, depth, [tuple(v >> l for v in s_) for s_ in surf])
        scale = float(rhs.abs().max()) * hs[l] * hs[l]
        e0 = rand(n, 0.1 * scale)
        for zf in (0, 1):
            e1 = e0.clone()
            _lib.check(lib.casmvs_poisson_smooth(_ptr(e1), _ptr(rhs), n, l, hs[l], 1, zf, st), "smooth")
            _record(depth, F.check_smooth(e0.view(n, n, n), e1.view(n, n, n), rhs.view(n, n, n), n, l,
                                          hs[l], wl, zero_first=bool(zf)))
            del e1
        out = torch.empty_like(e0)
        _lib.check(lib.casmvs_poisson_mg_residual(_ptr(e0), _ptr(rhs), n, l, hs[l], _ptr(out), st),
                   "mg_residual")
        _record(depth, F.check_mg_residual(e0.view(n, n, n), rhs.view(n, n, n), out.view(n, n, n), n, l,
                                           hs[l], wl))
        if l + 1 == len(sizes):
            break
        nc = n // 2
        c = torch.empty(nc ** 3, dtype=torch.float32, device=DEV)
        _lib.check(lib.casmvs_poisson_restrict(_ptr(out), n, _ptr(c), st), "restrict")
        wc = _wins(nc, depth, [tuple(v >> (l + 1) for v in s_) for s_ in surf])
        _record(depth, F.check_restrict(out.view(n, n, n), c.view(nc, nc, nc), n, l + 1, wc))
        del out
        ec = rand(nc, 0.1 * scale)
        f1 = e0.clone()
        _lib.check(lib.casmvs_poisson_prolong_add(_ptr(ec), nc, _ptr(f1), l, st), "prolong_add")
        _record(depth, F.check_prolong_add(ec.view(nc, nc, nc), e0.view(n, n, n), f1.view(n, n, n), nc, l,
                                           wl))
        del f1, ec, e0
        rhs = c
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [6, 7, 8, 9, 10])
def test_kernels_at_every_level(depth):
    N = 1 << depth
    need = 60 * N ** 3 + (1 << 30)                 # chi, b, r, V, W, C and the level fields
    budget = mesh.device_budget(torch.device(DEV))
    assert budget >= need, f"depth {depth} needs {need / 2**30:.1f} GiB, {budget / 2**30:.1f} free"
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    _level_kernels(depth, None)
    dt = time.perf_counter() - t0
    print(f"\n[poisson-fp64] depth {depth} per-kernel checks ran: {dt:.1f} s, peak "
          f"{torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------- whole pipeline
def _stage_checks(c, depth, windowed=False):
    """poisson_mesh with fields= against float64, every stage."""
    xyz, rgb, nrm, cams = _cuda(c["xyz"]), _cuda(c["rgb"]), _cuda(c["normals"]), c["cams"]
    got = {}
    _, _, faces, st = poisson.poisson_mesh(xyz, rgb, nrm, cams, depth=depth, fields=got)
    g = poisson.grid(xyz, depth)
    N, h, lo = g["N"], g["h"], g["lo"]
    # cells and normals through the ABI on the same cloud, as poisson_mesh sorts them
    keys, unit = _keys(xyz, nrm, g)
    r1, r2 = F.check_cell_keys(xyz, nrm, h, lo, N, keys, unit)
    _record(depth, r1, *([r2] if r2 is not None else []))
    skeys, perm = torch.sort(keys, stable=True)
    ok = skeys != F.KEY_NONE
    skeys, perm = skeys[ok], perm[ok]
    p = xyz[perm].contiguous()
    if nrm is None:
        lib = _lib.load()
        cells, counts, start = poisson._cells(skeys)
        cell_of = poisson._cell_map(cells, N)
        mom = torch.empty(len(cells), 10, dtype=torch.float64, device=DEV)
        _lib.check(lib.casmvs_poisson_cell_moments(_ptr(p), _ptr(start), len(cells), *g["centre"],
                                                   _ptr(mom), _st()), "moments")
        _record(depth, F.check_moments(p, start, g["centre"], mom))
        cn = torch.empty(len(cells), 3, dtype=torch.float64, device=DEV)
        cok = torch.empty(len(cells), dtype=torch.uint8, device=DEV)
        _lib.check(lib.casmvs_poisson_cell_normals(_ptr(cells), _ptr(cell_of), _ptr(mom), len(cells), N,
                                                   _ptr(cn), _ptr(cok), _st()), "normals")
        rep = F.check_normals(cells, mom, N, cn, cok)
        assert rep.exempt <= max(10, len(cells) // 100), rep.describe()
        _record(depth, rep)
        pcell = torch.repeat_interleave(torch.arange(len(cells), dtype=torch.int32, device=DEV), counts)
        out = torch.empty(len(p), 3, dtype=torch.float32, device=DEV)
        camd = torch.as_tensor(cams, dtype=torch.float64, device=DEV)
        _lib.check(lib.casmvs_poisson_orient(_ptr(p), _ptr(pcell), _ptr(cn), len(p), _ptr(camd),
                                             len(cams), _ptr(out), _st()), "orient")
        _record(depth, F.check_orient(p, pcell, cn, cams, out))
        kept = cok.bool()[pcell]
        want_idx, want_n = perm[kept], out[kept]
    else:
        want_idx, want_n = perm, unit[perm]
    assert torch.equal(got["index"], want_idx)
    assert torch.equal(got["normals"], want_n)
    pk = xyz[got["index"]].contiguous()
    col = rgb[got["index"]] if rgb is not None else None
    wins = F.windows(N, 32, _surface_nodes(pk.cpu().numpy(), g)) if windowed else None
    V, W, C = got["V"].view(N, N, N, 3), got["W"].view(N, N, N), got["C"].view(N, N, N, 3)
    _record(depth, *F.check_splat(pk, got["normals"], col, h, lo, N, V, W, C, wins).values())
    b = got["b"].view(N, N, N)
    _record(depth, F.check_rhs(V, b, N, h, wins))
    keep = got["keep"].view(N, N, N)
    _record(depth, F.check_trim(W, keep, N, wins))
    b0 = [v // 8 for v in lo]
    nbk = [(v + N - 1) // 8 - v // 8 + 1 for v in lo]
    flags = torch.zeros(nbk, dtype=torch.uint8, device=DEV)
    bk = got["keys"]
    B = 1 << 20
    bi = torch.stack([(bk >> 42) - B, ((bk >> 21) & 0x1FFFFF) - B, (bk & 0x1FFFFF) - B], 1)
    bi = bi - torch.tensor(b0, device=DEV)
    flags[bi[:, 0], bi[:, 1], bi[:, 2]] = 1
    _record(depth, F.check_brick_flags(keep, N, lo, b0, nbk, flags))
    chi = got["chi"].view(N, N, N)
    iso = got["iso"]
    _record(depth, *F.check_fill(bk, keep, W, C, chi, iso, got["weight"], got["color"], got["tsdf"], N,
                                 lo, wins).values())
    rep, rep_sum = F.check_iso(got["chi"], pk, h, lo, N, iso * len(pk))
    _record(depth, rep, rep_sum)
    # the solve: float64 residual of the kernel's chi, and the float64 multigrid's cycles
    r = b.double() - F.laplacian(chi, h)
    r = torch.where(F.interior(F.full(N), N, 0, DEV), r, 0.0)
    ratio64 = float(torch.linalg.vector_norm(r) / torch.linalg.vector_norm(b.double()))
    assert ratio64 <= poisson.TOL * 1.001, ratio64
    if not windowed:
        chi64, want = F.multigrid64(b, h)
        assert F.contraction_ok(st["ratios"], want), (st["ratios"], want)
        assert abs(st["cycles"] - (len(want) - 1)) <= 1
        assert (chi - chi64).abs().max() <= 1e-4 * chi64.abs().max()
        print(f"\n[poisson-fp64] depth {depth}: contraction per cycle "
              + " ".join(f"{a / b_:.3f}/{c_ / d:.3f}" for a, b_, c_, d in
                         zip(st["ratios"][1:], st["ratios"], want[1:], want)) + " (kernel/float64)")
    assert len(faces) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name,depth", [(n, d) for n, s in CASES.items() for d in s["depths"]])
def test_pipeline_stages(name, depth):
    _stage_checks(cloud(name), depth)


@pytest.mark.gpu
def test_pipeline_stages_depth_9_windowed():
    c = cloud("lo_mixed")
    _stage_checks(c, 9, windowed=True)


@pytest.mark.gpu
def test_depth_10_end_to_end():
    p, n = O.sphere(2_000_000, seed=9)
    need = poisson._bytes_needed(10, len(p))
    budget = mesh.device_budget(torch.device(DEV))
    assert budget >= need, f"depth 10 needs {need / 2**30:.1f} GiB, {budget / 2**30:.1f} free"
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    pd, nd = _cuda(p), _cuda(n)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    v, _, f, st = poisson.poisson_mesh(pd, normals=nd, depth=10)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f"\n[poisson-fp64] depth 10 end to end ran: {dt:.2f} s, peak "
          f"{torch.cuda.max_memory_allocated() / 2**30:.2f} GiB, {st['cycles']} cycles, "
          f"ratios {['%.2g' % r for r in st['ratios']]}")
    v, f = v.cpu().numpy(), f.cpu().numpy()
    d = np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - 1.0)
    assert st["residual"] <= poisson.TOL and st["dropped"] == 0
    assert d.max() < st["h"]
    assert M.is_closed_oriented(f) and M.euler_characteristic(len(v), f) == 2
