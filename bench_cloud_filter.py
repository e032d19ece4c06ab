"""Time statistical outlier removal on the GPU (cloud_filter.py, csrc/pcd_eval.cu) and measure what
it does to the scores of synthetic scenes.

1. Speed: bench_mesh.py's clouds (synth_scenes.sphere_scene, 49 and 150 views of 1152x864: every
   pixel that sees the scene, 34.2 M and 103.3 M points) at k = 20 and 64, std ratio 2.  Each
   phase (bounds and keys, sort and cells, search, statistics) is timed by a host clock around
   work that ends in a device synchronise, median of --repeats after one untimed run.  Also the
   peak device allocation above the input cloud per point (it sets BYTES_PER_POINT) and the
   search throughput in points/s; for scale, the float64 oracle's host time on 1 M of the points.
2. Effect, at the defaults (k = 20, std ratio 2), before and after filtering:
   - DTU accuracy, completeness and overall of synth_dtu.make_scene at outlier_frac 0.02 and 0.1;
   - the shares of points within tau of the analytic surface (accuracy) and of surface samples
     within tau of a point (completeness), tau = 1, 2, on bench_fusion.py's 60-view and thinned
     12-view sphere scenes, under both fusion rules;
   - precision, recall and F-score of synth_tnt.make_scene.
Prints one JSON line per row with the card name and power limit read in the same run.

    python bench_cloud_filter.py [--views 49 150] [--ks 20 64] [--repeats 3]
"""
import argparse
import json
import statistics
import tempfile
import time

import torch

import bench_fusion
from bench_mesh import card
from casmvsnet_pl_b200 import cloud_filter, dtu_eval, fusion, synth_dtu, synth_scenes, synth_tnt, tnt_eval

PHASES = ("bounds_keys_s", "sort_cells_s", "search_s", "statistics_s")


def speed(views, ks, repeats, name, power, dev):
    scene = synth_scenes.sphere_scene(views, (1152, 864), seed=0, device=dev)
    xyz = torch.cat([v["points"].to(dev) for v in scene]).float().contiguous()
    del scene
    torch.cuda.empty_cache()
    n = len(xyz)
    for k in ks:
        cloud_filter.remove_statistical_outliers(xyz, k)                   # warm-up
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        runs = []
        for _ in range(repeats):
            _, st = cloud_filter.remove_statistical_outliers(xyz, k)
            runs.append(st)
        peak = torch.cuda.max_memory_allocated() - base
        t = {p: statistics.median(r["time_s"][p] for r in runs) for p in PHASES}
        total = statistics.median(sum(r["time_s"][p] for p in PHASES) for r in runs)
        st = runs[0]
        print(json.dumps(dict(bench="speed", views=views, points=n, k=k, kept=st["kept"],
                              cell=st["cell"], cells=st["cells"], grid_trials=st["grid_trials"],
                              **{p[:-2] + "_ms": round(1e3 * v, 2) for p, v in t.items()},
                              total_ms=round(1e3 * total, 2),
                              search_points_per_s=round(n / t["search_s"]),
                              peak_bytes_per_point=round(peak / n, 1), repeats=repeats, gpu=name,
                              power_limit=power)), flush=True)
    return xyz


def oracle_time(xyz, name, power):
    from oracle import cloud_filter_oracle as O
    sub = xyz[torch.randperm(len(xyz), generator=torch.Generator().manual_seed(0))[:1_000_000]
              .to(xyz.device)].cpu().numpy()
    t0 = time.perf_counter()
    O.remove_statistical_outliers(sub, 20, 2.0)
    print(json.dumps(dict(bench="oracle_host", points=len(sub), k=20,
                          seconds=round(time.perf_counter() - t0, 2), gpu=name, power_limit=power)),
          flush=True)


def dtu_effect(name, power, dev):
    for frac in (0.02, 0.1):
        with tempfile.TemporaryDirectory() as d:
            p = synth_dtu.make_scene(d, scan=1, n_stl=100_000, n_data=200_000, seed=0,
                                     outlier_frac=frac)
            xyz = torch.from_numpy(p).to(dev)
            pts, _, _ = cloud_filter.filter_points(xyz)
            for tag, cloud in (("before", xyz), ("after", pts)):
                r = dtu_eval.evaluate_scan(cloud, 1, d)
                print(json.dumps(dict(bench="effect_dtu", outlier_frac=frac, cloud=tag,
                                      points=len(cloud), acc=round(r["acc"], 4),
                                      comp=round(r["comp"], 4), overall=round(r["overall"], 4),
                                      gpu=name, power_limit=power)), flush=True)


def fusion_effect(n_views, label, taus, name, power, dev):
    views = synth_scenes.sphere_scene(n_views, (1152, 864), seed=4, radius=bench_fusion.RADIUS,
                                      device=dev)
    metas, depths, probas, images, proj = bench_fusion.scan_inputs(views, 10, 7, dev)
    surf = torch.cat([v["points"].to(dev) for v in views])
    surf = surf[torch.randperm(len(surf), generator=torch.Generator().manual_seed(0))[:4_000_000].to(dev)]
    lo = (surf.min(0).values - 10).double().cpu().numpy()
    hi = (surf.max(0).values + 10).double().cpu().numpy()
    for rule in fusion.RULES:
        xyz, _ = fusion.fuse_scan(metas, depths, probas, images, proj, conf=0.5, rule=rule)
        pts, _, _ = cloud_filter.filter_points(xyz)
        for tag, cloud in (("before", xyz), ("after", pts)):
            row = dict(bench="effect_fusion", scene=label, rule=rule, cloud=tag, points=len(cloud))
            err = bench_fusion.surface_distance(cloud)
            for tau in taus:
                comp = dtu_eval.capped_nn(surf.float().contiguous(), cloud.contiguous(), lo, hi,
                                          cap=4 * tau, cell=2 * tau)
                row[f"accuracy_share_tau{tau:g}"] = round(float((err <= tau).double().mean()), 4)
                row[f"completeness_share_tau{tau:g}"] = round(float((comp <= tau).double().mean()), 4)
            print(json.dumps(dict(row, gpu=name, power_limit=power)), flush=True)


def tnt_effect(name, power, dev):
    with tempfile.TemporaryDirectory() as d:
        sc = synth_tnt.make_scene(d, seed=0)
        v = dtu_eval.read_points(sc["ply"])
        xyz = torch.from_numpy(v).to(dev)
        pts, _, _ = cloud_filter.filter_points(xyz)
        for tag, cloud in (("before", xyz), ("after", pts)):
            r = tnt_eval.evaluate_scene(cloud, sc["run_dir"], sc["gt_dir"], sc["scene"], tau=sc["tau"],
                                        images=sc["images"])
            print(json.dumps(dict(bench="effect_tnt", cloud=tag, points=len(cloud),
                                  precision=round(r["precision"], 4), recall=round(r["recall"], 4),
                                  fscore=round(r["fscore"], 4), gpu=name, power_limit=power)),
                  flush=True)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", nargs="+", type=int, default=[49, 150])
    ap.add_argument("--ks", nargs="+", type=int, default=[20, 64])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--taus", nargs="+", type=float, default=[1.0, 2.0])
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_cloud_filter.py needs a GPU")
    dev = "cuda:0"
    name, power = card()
    for i, views in enumerate(a.views):
        xyz = speed(views, a.ks, a.repeats, name, power, dev)
        if i == 0:
            oracle_time(xyz, name, power)
        del xyz
        torch.cuda.empty_cache()
    dtu_effect(name, power, dev)
    fusion_effect(60, "sphere_60_views", a.taus, name, power, dev)
    fusion_effect(12, "sphere_12_views_thinned", a.taus, name, power, dev)
    tnt_effect(name, power, dev)


if __name__ == "__main__":
    main()
