"""Time Poisson meshing on the GPU (poisson.py) on bench_mesh.py's scene: a sphere on a plane
(synth_scenes.sphere_scene), its points taken from 49 and 150 depth maps of 1152x864 (about 34 M
and 103 M points), normals estimated and oriented toward the views' camera centres, at grid
depths 8, 9 and 10.  Each phase is timed with CUDA events (median of --repeats runs after one
untimed warm-up run): sort, cell moments, normals, splat, right-hand side, trim and bricks, solve
(with its cycle count; it includes the iso level), extraction.  Also timed: reading the cloud
back from a binary PLY (host clock, separately) and the TSDF mesher (mesh.py) on the same views.
A depth that does not fit is reported with its refusal.  Prints one JSON line per (size, depth)
and per size for the TSDF path, with the card name and power limit read in the same run.

    python bench_poisson.py [--views 49 150] [--depths 8 9 10] [--repeats 3]
"""
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


def run_once(xyz, cams, depth):
    events = []
    torch.cuda.synchronize()
    _, _, _, st = poisson.poisson_mesh(xyz, None, cam_centres=cams, depth=depth, events=events,
                                       log=None)
    torch.cuda.synchronize()
    ev = dict(events)
    order = ["start"] + PHASES
    ms = {p: ev[order[i]].elapsed_time(ev[p]) for i, p in enumerate(PHASES, 0)}
    ms["total"] = ev["start"].elapsed_time(ev["extract"])
    return ms, st


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", nargs="+", type=int, default=[49, 150])
    ap.add_argument("--depths", nargs="+", type=int, default=[8, 9, 10])
    ap.add_argument("--wh", nargs=2, type=int, default=[1152, 864])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
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
        del xyz
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
