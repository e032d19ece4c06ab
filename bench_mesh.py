"""Time meshing on the GPU: brick allocation, TSDF integration and marching-cubes extraction of
an analytic scene (a sphere on a plane, synth_scenes.sphere_scene, depth maps rendered from a
seed) at the sizes a user runs: 49 and 150 views of 1152x864.  Each phase is timed with CUDA
events and ends in a synchronise; one full untimed run per size comes first (warm-up).  Prints
one JSON line per size with the card name and power limit read in the same run.

    python bench_mesh.py [--views 49 150] [--wh 1152 864] [--repeats 3]
"""
import argparse
import json
import subprocess

import numpy as np
import torch

from casmvsnet_pl_b200 import mesh, synth_scenes


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def run_once(views, voxel):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    torch.cuda.synchronize()
    ev[0].record()
    vol = mesh.TSDFVolume([v["points"] for v in views], voxel)
    ev[1].record()
    vol.integrate([v["depth"] for v in views], [v["image"] for v in views], [v["P"] for v in views])
    ev[2].record()
    verts, cols, faces = vol.extract()
    ev[3].record()
    torch.cuda.synchronize()
    ms = [ev[i].elapsed_time(ev[i + 1]) for i in range(3)]
    return ms, dict(bricks=vol.n_bricks, voxels=vol.n_voxels, vertices=len(verts),
                    triangles=len(faces), dropped=vol.dropped)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", nargs="+", type=int, default=[49, 150])
    ap.add_argument("--wh", nargs=2, type=int, default=[1152, 864])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh.py needs a GPU")
    name, power = card()
    for n in a.views:
        views = synth_scenes.sphere_scene(n, tuple(a.wh), seed=a.seed, device="cuda:0")
        voxel = mesh.default_voxel_size([v["depth"] for v in views], [v["P"] for v in views])
        n_points = sum(len(v["points"]) for v in views)
        run_once(views, voxel)                                   # warm-up
        times = []
        for _ in range(a.repeats):
            ms, stats = run_once(views, voxel)
            times.append(ms)
        med = np.median(np.array(times), axis=0)
        print(json.dumps(dict(views=n, wh=a.wh, points=n_points, voxel=voxel, **stats,
                              alloc_ms=round(float(med[0]), 3), integrate_ms=round(float(med[1]), 3),
                              extract_ms=round(float(med[2]), 3),
                              total_ms=round(float(med.sum()), 3), repeats=a.repeats,
                              gpu=name, power_limit=power)), flush=True)
        del views
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
