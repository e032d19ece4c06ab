"""Time mesh cleaning on the GPU (mesh_clean.py) on the meshes bench_simplify.py decimates: the
49-view TSDF mesh of the sphere-on-a-plane scene (synth_scenes.sphere_scene) and Poisson meshes of
the same scene's points at depths 9 and 10.  Per mesh: the time of each phase (cleanup, pieces,
areas, loops, triangulation, compaction) from CUDA events, median of --repeats runs after one
untimed warm-up, torch's peak allocation, pieces removed and holes filled or skipped.

Then two effects of cleaning: whether the cleaned TSDF mesh lets simplification reach its 1 %
target, against the uncleaned mesh; and the DTU accuracy and completeness (dtu_eval.evaluate_mesh)
of the Poisson mesh of synth_dtu scenes with more or fewer outliers and holes, before and after
cleaning.  Prints one JSON line per row with the card name and power limit read in the same run.

    python bench_mesh_clean.py [--views 49] [--wh 1152 864] [--depths 9 10] [--max_hole 128]
"""
import argparse
import json
import tempfile

import numpy as np
import torch

from bench_mesh import card
from casmvsnet_pl_b200 import dtu_eval, mesh, mesh_clean, poisson, simplify, synth_dtu, synth_scenes

PHASES = ("cleanup", "pieces", "areas", "loops", "triangulation", "compaction")


def run_once(v, c, f, min_ratio, max_hole):
    """mesh_clean.clean_mesh's steps with an event between phases -> ms per phase."""
    ev = lambda: torch.cuda.Event(enable_timing=True)      # noqa: E731
    marks = []

    def mark(name):
        e = ev()
        e.record()
        marks.append((name, e))

    torch.cuda.synchronize()
    mark("start")
    fc, _ = mesh_clean.cleanup(v, f)
    mark("cleanup")
    pc = mesh_clean.pieces(v, fc, mark=mark)
    keep_piece = pc["count"] >= mesh_clean.piece_threshold(pc["count"], 0, min_ratio)
    keep = keep_piece[pc["piece"]]
    fc = fc[keep].contiguous()
    mark("areas")
    lp = mesh_clean.boundary_loops(fc, len(v))
    small = lp["sizes"] <= max_hole
    mark("loops")
    status, _, tris, row = mesh_clean.fill_holes(v, lp, lp["owners"][small], lp["sizes"][small],
                                                 pc["area"][pc["piece"][keep]])
    fc = torch.cat([fc, tris[status[row] == mesh_clean.STATUS_FILLED]])
    mark("triangulation")
    simplify._compact(v, c, fc)
    mark("compaction")
    torch.cuda.synchronize()
    return {name: a.elapsed_time(b) for (_, a), (name, b) in zip(marks, marks[1:])}


def bench(label, v, c, f, a, name, power):
    kw = dict(min_ratio=a.min_ratio, max_hole=a.max_hole)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    V, C, F, st = mesh_clean.clean_mesh(v, c, f, **kw)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del V, C, F
    run_once(v, c, f, a.min_ratio, a.max_hole)                            # warm-up
    rows = [run_once(v, c, f, a.min_ratio, a.max_hole) for _ in range(a.repeats)]
    med = {k: float(np.median([x[k] for x in rows])) for k in PHASES}
    tot = float(np.median([sum(x.values()) for x in rows]))
    print(json.dumps(dict(mesh=label, vertices_in=len(v), **kw, **st, total_ms=round(tot, 2),
                          **{k + "_ms": round(x, 3) for k, x in med.items()},
                          peak_alloc_mib=round(peak / 2 ** 20, 1),
                          peak_bytes_per_face=round(peak / len(f), 1),
                          peak_bytes_needed=len(f) * mesh_clean.BYTES_PER_FACE
                          + len(v) * mesh_clean.BYTES_PER_VERTEX,
                          repeats=a.repeats, gpu=name, power_limit=power)), flush=True)
    return st


def simplify_effect(label, v, c, f, a, name, power):
    """Simplification to 1 % of the input faces, before and after cleaning."""
    target = max(1, round(0.01 * len(f)))
    out = dict(mesh=label, target=target)
    _, _, _, s0 = simplify.simplify_mesh(v, c, f, target, log=lambda m: None)
    V, C, F, _ = mesh_clean.clean_mesh(v, c, f, min_ratio=a.min_ratio, max_hole=a.max_hole)
    _, _, _, s1 = simplify.simplify_mesh(V, C, F, target, log=lambda m: None)
    out.update(raw_faces=s0["faces"], raw_stop=s0["stop"], cleaned_faces_in=len(F),
               cleaned_faces=s1["faces"], cleaned_stop=s1["stop"], gpu=name, power_limit=power)
    print(json.dumps(out), flush=True)


def score_effect(a, name, power):
    """DTU scores of a synth_dtu scene's Poisson mesh before and after cleaning."""
    cams = synth_dtu.CENTER + np.array([[0, 0, -500.0], [80, 0, -480], [-80, 40, -490]])
    for outlier_frac, hole_frac in ((0.02, 0.1), (0.1, 0.1), (0.02, 0.3)):
        with tempfile.TemporaryDirectory() as gt:
            p = synth_dtu.make_scene(gt, scan=1, seed=a.seed, outlier_frac=outlier_frac,
                                     hole_frac=hole_frac)
            v, c, f, _ = poisson.poisson_mesh(torch.from_numpy(p).cuda(), cam_centres=cams,
                                              depth=a.dtu_depth, log=lambda m: None)
            raw = dtu_eval.evaluate_mesh((v, f), 1, gt)
            V, C, F, st = mesh_clean.clean_mesh(v, c, f, min_ratio=a.min_ratio, max_hole=a.max_hole)
            cl = dtu_eval.evaluate_mesh((V, F), 1, gt)
        print(json.dumps(dict(scene="synth_dtu", outlier_frac=outlier_frac, hole_frac=hole_frac,
                              poisson_depth=a.dtu_depth, faces=len(f), cleaned_faces=len(F),
                              pieces_removed=st["pieces_removed"], holes_filled=st["holes_filled"],
                              raw=dict(acc=raw["acc"], comp=raw["comp"],
                                       overall=raw["overall"]),
                              cleaned=dict(acc=cl["acc"], comp=cl["comp"],
                                           overall=cl["overall"]),
                              gpu=name, power_limit=power)), flush=True)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--wh", nargs=2, type=int, default=[1152, 864])
    ap.add_argument("--depths", nargs="*", type=int, default=[9, 10])
    ap.add_argument("--min_ratio", type=float, default=0.01)
    ap.add_argument("--max_hole", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--dtu_depth", type=int, default=9, help="Poisson depth of the DTU-like meshes "
                                                             "(0: skip the score rows)")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh_clean.py needs a GPU")
    name, power = card()
    views = synth_scenes.sphere_scene(a.views, tuple(a.wh), seed=a.seed, device="cuda:0")
    depths, images, Ps = [x["depth"] for x in views], [x["image"] for x in views], [x["P"] for x in views]
    pts = [x["points"] for x in views]
    v, c, f, _ = mesh.mesh_views(pts, depths, images, Ps)
    bench(f"tsdf_{a.views}views", v, c, f, a, name, power)
    simplify_effect(f"tsdf_{a.views}views", v, c, f, a, name, power)
    del v, c, f
    p = torch.cat(pts)
    rgb = torch.cat([x["image"][x["depth"] > 0] for x in views]).to(torch.uint8)
    cams = np.stack([-np.linalg.inv(P[:3, :3].astype(np.float64)) @ P[:3, 3] for P in Ps])
    del views, depths, images, pts
    torch.cuda.empty_cache()
    for d in a.depths:
        v, c, f, _ = poisson.poisson_mesh(p, rgb, cam_centres=cams, depth=d, log=lambda m: None)
        torch.cuda.empty_cache()
        bench(f"poisson_d{d}", v, c, f, a, name, power)
        del v, c, f
        torch.cuda.empty_cache()
    if a.dtu_depth:
        score_effect(a, name, power)


if __name__ == "__main__":
    main()
