"""Time Poisson meshing on the GPU (poisson.py) on bench_mesh.py's scene: a sphere on a plane
(synth_scenes.sphere_scene), its points taken from 49 and 150 depth maps of 1152x864 (about 34 M
and 103 M points), normals estimated and oriented toward the views' camera centres, at grid
depths 8, 9 and 10.  Each phase is timed with CUDA events (median of --repeats runs after one
untimed warm-up run): sort, cell moments, normals, splat, right-hand side, trim and bricks, solve
(with its cycle count; it includes the iso level), extraction.  Also timed: reading the cloud
back from a binary PLY (host clock, separately) and the TSDF mesher (mesh.py) on the same views.
A depth that does not fit is reported with its refusal.  Prints one JSON line per (size, depth)
and per size for the TSDF path, with the card name and power limit read in the same run.
With --point_weight A > 0, each (size, depth) also gets a screened row: the screen phase (moments
and the screened solve) and its cycle count, the peak memory beside the unscreened row's, and the
screened hot path on the finest level timed alone (CUDA events over SMOOTH_SWEEPS calls): one
smoother sweep, the float32 multigrid residual and the double residual, each with the bytes one
pass must move (per node its fields and mask, per surface node its stencil row) over that time.
A screened row's "solve" is the unscreened solve and its iso level; filling the bricks' tsdf,
which an unscreened row's "solve" includes, moves into "screen".

    python bench_poisson.py [--views 49 150] [--depths 8 9 10] [--repeats 3] [--point_weight 4]
"""
import ctypes
import argparse
import json
import os
import tempfile
import time

import numpy as np
import torch

from bench_mesh import card, run_once as tsdf_once
from casmvsnet_pl_b200 import _lib, fusion, mesh, poisson, synth_scenes

PHASES = ["sort", "moments", "normals", "splat", "rhs", "trim_bricks", "solve", "extract"]
SCREEN_PHASES = PHASES[:-1] + ["screen", "extract"]
SMOOTH_SWEEPS = 8
HBM_BYTES_PER_S = 3.35e12              # H100 SXM data sheet


def run_once(xyz, cams, depth, point_weight=0.0):
    events = []
    torch.cuda.synchronize()
    kw = dict(point_weight=point_weight) if point_weight > 0 else {}
    _, _, _, st = poisson.poisson_mesh(xyz, None, cam_centres=cams, depth=depth, events=events,
                                       log=None, **kw)
    torch.cuda.synchronize()
    ev = dict(events)
    phases = SCREEN_PHASES if point_weight > 0 else PHASES
    order = ["start"] + phases
    ms = {p: ev[order[i]].elapsed_time(ev[p]) for i, p in enumerate(phases, 0)}
    ms["total"] = ev["start"].elapsed_time(ev["extract"])
    return ms, st


def smoother_rate(xyz, depth, point_weight):
    """The screened hot path on the finest level, built from every point of the cloud: CUDA-event
    times of SMOOTH_SWEEPS smoother sweeps, one float32 multigrid residual and one double residual,
    each with the bytes one pass must move -> dict."""
    g = poisson.grid(xyz, depth)
    N, h = g["N"], g["h"]
    levels = poisson._screen_levels(xyz, N, h, g["lo"])
    lv = levels[0]
    del levels
    gg = point_weight * len(lv["keys"]) / len(xyz)
    ns = len(lv["stencil"])
    dev = xyz.device
    r = torch.zeros(N ** 3, dtype=torch.float32, device=dev)
    e = torch.zeros_like(r)
    out = torch.empty_like(r)
    lib, st_ = _lib.load(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = poisson._ptr
    ops = (P(lv["mask"]), P(lv["srow"]), P(lv["stencil"]), N, 0, h, gg)

    def timed(fn, k):
        fn()                                                         # warm-up
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(k):
            fn()
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / k
    res = {}
    ms = timed(lambda: _lib.check(lib.casmvs_poisson_screen_smooth(P(e), P(r), *ops, 1, 0, st_),
                                  "smooth"), SMOOTH_SWEEPS)
    res["smooth"] = (ms, N ** 3 * (4 + 4 + 4 + 1) + ns * (4 + 27 * 4))   # e, e', r, mask; srow, stencil
    ms = timed(lambda: _lib.check(lib.casmvs_poisson_screen_mg_residual(P(e), P(r), *ops, P(out), st_),
                                  "mg_residual"), SMOOTH_SWEEPS)
    res["mg_residual"] = (ms, N ** 3 * (4 + 4 + 1 + 4) + ns * (4 + 27 * 4))
    del e
    chi = torch.zeros(N ** 3, dtype=torch.float64, device=dev)
    ws = torch.empty(lib.casmvs_poisson_workspace_bytes(N ** 3) // 8, dtype=torch.float64, device=dev)
    rr = torch.zeros(1, dtype=torch.float64, device=dev)
    ms = timed(lambda: _lib.check(lib.casmvs_poisson_screen_residual(
        P(chi), P(r), P(lv["mask"]), P(lv["srow"]), P(lv["stencil64"]), N, h, gg, P(out), P(ws),
        P(rr), st_), "residual"), SMOOTH_SWEEPS)
    res["residual"] = (ms, N ** 3 * (8 + 4 + 1 + 4) + ns * (4 + 27 * 8))
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", nargs="+", type=int, default=[49, 150])
    ap.add_argument("--depths", nargs="+", type=int, default=[8, 9, 10])
    ap.add_argument("--wh", nargs=2, type=int, default=[1152, 864])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--point_weight", type=float, default=0.0,
                    help="also time screened Poisson at this point weight (> 0)")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_poisson.py needs a GPU")
    name, power = card()
    for n in a.views:
        views = synth_scenes.sphere_scene(n, tuple(a.wh), seed=a.seed, device="cuda:0")
        cams = np.stack([-np.linalg.inv(v["P"][:3, :3].astype(np.float64)) @ v["P"][:3, 3] for v in views])
        xyz = torch.cat([v["points"] for v in views])
        n_points = len(xyz)
        with tempfile.TemporaryDirectory() as d:         # the PLY read, host clock
            path = os.path.join(d, "cloud.ply")
            fusion.write_ply(path, xyz, torch.full_like(xyz, 128, dtype=torch.uint8))
            t0 = time.perf_counter()
            host = poisson.read_cloud(path)
            read_s = time.perf_counter() - t0
            del host
        voxel = mesh.default_voxel_size([v["depth"] for v in views], [v["P"] for v in views])
        tsdf_once(views, voxel)
        t = np.median(np.array([tsdf_once(views, voxel)[0] for _ in range(a.repeats)]), axis=0)
        print(json.dumps(dict(method="tsdf", views=n, points=n_points, voxel=voxel,
                              alloc_ms=round(float(t[0]), 3), integrate_ms=round(float(t[1]), 3),
                              extract_ms=round(float(t[2]), 3), total_ms=round(float(t.sum()), 3),
                              gpu=name, power_limit=power)), flush=True)
        del views
        torch.cuda.empty_cache()
        for depth in a.depths:
            row = dict(method="poisson", views=n, points=n_points, depth=depth,
                       ply_read_s=round(read_s, 3), gpu=name, power_limit=power)
            torch.cuda.reset_peak_memory_stats()
            try:
                run_once(xyz, cams, depth)                           # warm-up
                runs = []
                for _ in range(a.repeats):
                    torch.cuda.empty_cache()         # each run starts from the same free memory
                    runs.append(run_once(xyz, cams, depth))
            except _lib.CasMVSError as e:
                row["refused"] = str(e)
                print(json.dumps(row), flush=True)
                continue
            st = runs[-1][1]
            for p in PHASES + ["total"]:
                row[f"{p}_ms"] = round(float(np.median([r[0][p] for r in runs])), 3)
            row.update(cycles=st["cycles"], residual=st["residual"], dropped=st["dropped"],
                       bricks=st["bricks"], vertices=st["vertices"], triangles=st["triangles"],
                       peak_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                       repeats=a.repeats)
            print(json.dumps(row), flush=True)
            torch.cuda.empty_cache()
            if a.point_weight > 0:
                screened_row(a, xyz, cams, depth, n, n_points, name, power, row["peak_gib"])
        del xyz
        torch.cuda.empty_cache()


def screened_row(a, xyz, cams, depth, n, n_points, name, power, peak0):
    row = dict(method="poisson", point_weight=a.point_weight, views=n, points=n_points, depth=depth,
               gpu=name, power_limit=power, unscreened_peak_gib=peak0)
    torch.cuda.reset_peak_memory_stats()
    try:
        run_once(xyz, cams, depth, a.point_weight)                    # warm-up
        runs = []
        for _ in range(a.repeats):
            torch.cuda.empty_cache()
            runs.append(run_once(xyz, cams, depth, a.point_weight))
    except _lib.CasMVSError as e:
        row["refused"] = str(e)
        print(json.dumps(row), flush=True)
        torch.cuda.empty_cache()
        return
    st = runs[-1][1]
    for p in SCREEN_PHASES + ["total"]:
        row[f"{p}_ms"] = round(float(np.median([r[0][p] for r in runs])), 3)
    row.update(cycles=st["cycles"], screened_cycles=st["screened_cycles"],
               screened_residual=st["screened_ratios"][-1], vertices=st["vertices"],
               triangles=st["triangles"],
               peak_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), repeats=a.repeats)
    torch.cuda.empty_cache()
    for k, (ms, nbytes) in smoother_rate(xyz, depth, a.point_weight).items():
        row.update({f"{k}_ms": round(ms, 3), f"{k}_bytes": nbytes,
                    f"{k}_tb_per_s": round(nbytes / (ms * 1e-3) / 1e12, 3),
                    f"{k}_of_hbm": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)})
    print(json.dumps(row), flush=True)
    torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
