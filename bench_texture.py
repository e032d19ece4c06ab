"""Time mesh texturing on the GPU (texture.py) on bench_mesh.py's scene: a sphere on a plane seen by
49 views of 1152x864 (synth_scenes.sphere_scene), its full TSDF mesh and that mesh decimated to
10 % and 1 % (simplify.py).  The photos are the scene's images rounded to uint8 once.  Each phase
is timed with CUDA events (the host phases with a host clock after a synchronise) in a run that
follows one untimed warm-up run of the same mesh.  Prints one JSON line per mesh with the charts
at R = 0 and R = 4 smoothing rounds, the pages, the packed share, the peak allocation above what
the mesh and photos hold, and the card name and power limit read in the same run.

    python bench_texture.py [--views 49] [--wh 1152 864] [--ratios 1 0.1 0.01] [--out DIR]
"""
import argparse
import json
import os
import tempfile
import time

import numpy as np
import torch

from bench_mesh import card
from casmvsnet_pl_b200 import mesh, simplify, synth_scenes, texture

PHASES = ("keys", "scores", "smooth", "charts", "pack", "fill")


def run_once(v, c, f, photos, Ps, out_dir):
    evs = []

    def mark(phase):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        evs.append((phase, e, time.perf_counter()))
        if phase == "charts":                        # packing is host work: clock it on the host
            torch.cuda.synchronize()
            evs[-1] = (phase, e, time.perf_counter())

    torch.cuda.synchronize()
    start = torch.cuda.Event(enable_timing=True)
    start.record()
    uv, page, atlas, st = texture.texture_mesh(v, c, f, photos, Ps, mark=mark)
    torch.cuda.synchronize()
    ms = dict.fromkeys(PHASES, 0.0)
    prev, prev_t = start, None
    for phase, e, t in evs:
        if phase == "pack":
            ms[phase] += (t - prev_t) * 1e3
        else:
            ms[phase] += prev.elapsed_time(e)
        prev, prev_t = e, t
    t0 = time.perf_counter()
    texture.write_textured_obj(os.path.join(out_dir, "bench.obj"), v, f, uv, page, atlas)
    ms["write_obj_png"] = (time.perf_counter() - t0) * 1e3
    return ms, st


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--wh", nargs=2, type=int, default=[1152, 864])
    ap.add_argument("--ratios", nargs="+", type=float, default=[1.0, 0.1, 0.01])
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="where the OBJ / PNG files go (default: a "
                                                "temporary directory)")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_texture.py needs a GPU")
    name, power = card()
    views = synth_scenes.sphere_scene(a.views, tuple(a.wh), seed=a.seed, device="cuda:0")
    voxel = mesh.default_voxel_size([x["depth"] for x in views], [x["P"] for x in views])
    v0, c0, f0, _ = mesh.mesh_views([x["points"] for x in views], [x["depth"] for x in views],
                                    [x["image"] for x in views], [x["P"] for x in views], voxel)
    photos = [x["image"].round().clamp(0, 255).to(torch.uint8) for x in views]
    Ps = [x["P"] for x in views]
    del views
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as tmp:
        out_dir = a.out or tmp
        os.makedirs(out_dir, exist_ok=True)
        for r in a.ratios:
            if r < 1:
                v, c, f, _ = simplify.simplify_mesh(v0, c0, f0, max(1, round(r * len(f0))))
            else:
                v, c, f = v0, c0, f0
            run_once(v, c, f, photos, Ps, out_dir)                       # warm-up
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            ms, st = run_once(v, c, f, photos, Ps, out_dir)
            peak = torch.cuda.max_memory_allocated() - base
            r0 = st["charts_unsmoothed"]
            print(json.dumps(dict(views=len(Ps), wh=a.wh, ratio=r, faces=len(f), voxel=voxel,
                                  **{f"{k}_ms": round(val, 3) for k, val in ms.items()},
                                  gpu_total_ms=round(sum(ms[k] for k in PHASES if k != "pack"), 3),
                                  peak_alloc_mib=round(peak / 2**20, 1),
                                  charts_r0=r0, charts_r4=st["charts"], flat_charts=st["flat_charts"],
                                  unseen_faces=st["unseen_faces"],
                                  candidates_per_face=round(st["candidates_per_face"], 3),
                                  pages=st["pages"], page_side=st["page_side"],
                                  packed_share=round(st["packed_share"], 4),
                                  gpu=name, power_limit=power)), flush=True)
            del v, c, f
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
