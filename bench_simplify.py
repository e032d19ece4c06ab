"""Time mesh simplification on the GPU (simplify.py) on the meshes a user gets from the meshers:
bench_mesh.py's 49-view TSDF mesh of the sphere-on-a-plane scene (synth_scenes.sphere_scene) and
Poisson meshes of the same scene's points at depths 9 and 10, each decimated to 10 % and 1 % of
its faces.  Per size: rounds, total time and the time of each phase (edges + CSR, costs and
validity, selection, collapse + compaction) from CUDA events, median of --repeats runs after one
untimed warm-up, and torch's peak allocation.  The serial greedy decimation of
oracle/simplify_oracle.py is timed on the host at about 100 k faces, for scale.  Prints one JSON
line per row with the card name and power limit read in the same run.

    python bench_simplify.py [--views 49] [--wh 1152 864] [--depths 9 10] [--ratios 0.1 0.01]
"""
import argparse
import json
import time

import numpy as np
import torch

from bench_mesh import card
from casmvsnet_pl_b200 import mesh, poisson, simplify, synth_scenes

PHASES = ("prepare", "edges_csr", "costs", "select", "collapse", "compact")


def run_once(v, c, f, target):
    """simplify.simplify_mesh's loop with an event between phases -> (ms per phase, stats)."""
    ms = dict.fromkeys(PHASES, 0.0)
    ev = lambda: torch.cuda.Event(enable_timing=True)      # noqa: E731
    pairs = []

    def mark(name, e0):
        e1 = ev()
        e1.record()
        pairs.append((name, e0, e1))
        return e1

    torch.cuda.synchronize()
    e = ev()
    e.record()
    P, C, fc, frozen, Q, dropped = simplify._prepare(v, c, f)
    e = mark("prepare", e)
    rounds = 0
    while len(fc) > target:
        topo = simplify._topology(fc, len(P))
        e = mark("edges_csr", e)
        st = simplify._edge_costs(P, Q, fc, frozen, None, topo)
        e = mark("costs", e)
        sel, thr = simplify._select(st, fc, len(P))
        if sel is None:
            break
        idx = simplify._budget(st, sel, len(fc), target)
        e = mark("select", e)
        fc = simplify._collapse(P, C, Q, fc, st, idx)
        e = mark("collapse", e)
        rounds += 1
    V, Cc, F = simplify._compact(P, C, fc)
    mark("compact", e)
    torch.cuda.synchronize()
    for name, a, b in pairs:
        ms[name] += a.elapsed_time(b)
    return ms, dict(rounds=rounds, faces_out=len(F), vertices_out=len(V))


def bench(label, v, c, f, ratios, repeats, name, power):
    for r in ratios:
        target = max(1, round(r * len(f)))
        ref = simplify.simplify_mesh(v, c, f, target, log=lambda m: None)[3]
        run_once(v, c, f, target)                                         # warm-up
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        rows = [run_once(v, c, f, target) for _ in range(repeats)]
        peak = torch.cuda.max_memory_allocated() - base
        assert all(x[1]["faces_out"] == ref["faces"] for x in rows)
        med = {k: float(np.median([x[0][k] for x in rows])) for k in PHASES}
        tot = float(np.median([sum(x[0].values()) for x in rows]))
        print(json.dumps(dict(mesh=label, faces_in=len(f), vertices_in=len(v), target=target,
                              faces_out=ref["faces"], rounds=ref["rounds"], stop=ref["stop"],
                              total_ms=round(tot, 2), **{k + "_ms": round(x, 2) for k, x in med.items()},
                              peak_alloc_mib=round(peak / 2 ** 20, 1),
                              peak_bytes_per_face=round(peak / len(f), 1), repeats=repeats,
                              gpu=name, power_limit=power)), flush=True)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--wh", nargs=2, type=int, default=[1152, 864])
    ap.add_argument("--depths", nargs="*", type=int, default=[9, 10])
    ap.add_argument("--ratios", nargs="+", type=float, default=[0.1, 0.01])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--serial_grid", type=int, default=134,
                    help="grid of the host serial-greedy sphere (134: about 100 k faces; 0: skip)")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_simplify.py needs a GPU")
    name, power = card()
    views = synth_scenes.sphere_scene(a.views, tuple(a.wh), seed=a.seed, device="cuda:0")
    depths, images, Ps = [x["depth"] for x in views], [x["image"] for x in views], [x["P"] for x in views]
    pts = [x["points"] for x in views]
    v, c, f, _ = mesh.mesh_views(pts, depths, images, Ps)
    bench(f"tsdf_{a.views}views", v, c, f, a.ratios, a.repeats, name, power)
    del v, c, f
    p = torch.cat(pts)
    rgb = torch.cat([x["image"][x["depth"] > 0] for x in views]).to(torch.uint8)
    cams = np.stack([-np.linalg.inv(P[:3, :3].astype(np.float64)) @ P[:3, 3] for P in Ps])
    del views, depths, images, pts
    torch.cuda.empty_cache()
    for d in a.depths:
        v, c, f, _ = poisson.poisson_mesh(p, rgb, cam_centres=cams, depth=d, log=lambda m: None)
        torch.cuda.empty_cache()
        bench(f"poisson_d{d}", v, c, f, a.ratios, a.repeats, name, power)
        del v, c, f
        torch.cuda.empty_cache()
    if a.serial_grid:
        from oracle import simplify_oracle as S
        v, c, f = S.sphere_mesh(a.serial_grid)
        t = time.perf_counter()
        Vs, _, Fs = S.serial_simplify(v, c, f, len(f) // 10)
        host_s = time.perf_counter() - t
        V, C, F, st = simplify.simplify_mesh(torch.from_numpy(v).cuda(), torch.from_numpy(c).cuda(),
                                             torch.from_numpy(f).cuda(), len(f) // 10)
        torch.cuda.synchronize()
        t = time.perf_counter()
        simplify.simplify_mesh(torch.from_numpy(v).cuda(), torch.from_numpy(c).cuda(),
                               torch.from_numpy(f).cuda(), len(f) // 10)
        torch.cuda.synchronize()
        gpu_s = time.perf_counter() - t
        err = lambda x: float(np.abs(np.linalg.norm(np.asarray(x, np.float64), axis=1) - 1).mean())  # noqa: E731
        print(json.dumps(dict(mesh=f"sphere_grid{a.serial_grid}", faces_in=len(f), target=len(f) // 10,
                              serial_host_s=round(host_s, 2), serial_faces=len(Fs),
                              serial_mean_radial_error=err(Vs), gpu_s=round(gpu_s, 4),
                              gpu_rounds=st["rounds"], gpu_mean_radial_error=err(V.cpu().numpy()),
                              gpu=name, power_limit=power)), flush=True)


if __name__ == "__main__":
    main()
