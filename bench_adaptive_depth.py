"""Adaptive depth ranges (README "Adaptive depth ranges"): cascade time per depth map, uniform
against adaptive sampling, alternating in one process, at cfg2 (640x512, V = 3) and 1152x864
(V = 5), and per-kernel K1 / K3 / K4 device times from torch.profiler.  K1 may halve its depth
runs more often where a pixel's window is wide; the profiler rows show whether it costs time.
Prints one JSON line per row, with the card name and power limit read in the same run.

--study fine-tunes the network with the photometric loss on a synthetic textured capture, flat
(tilt 0) and sloped (tilt 2.25), once per sampling mode from the same random initialisation, and
reports at level 0 the mean |d - gt| in uniform-mode intervals and the share within 1, 2 and 4
intervals; and at stages 1 and 0 the coverage (share of pixels whose ground truth lies within
that stage's first and last plane) and the median plane spacing.

    python bench_adaptive_depth.py [--iters 30] [--rounds 3]
    python bench_adaptive_depth.py --study [--steps 128]
"""
import argparse
import json
import subprocess
import time

import torch

from casmvsnet_pl_b200 import ABN, synth
from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet

SIZES = {"cfg2": (640, 512, 3), "1152x864_V5": (1152, 864, 5)}
K1 = ("warp_var_smem", "warp_cost_kernel")
K3 = ("regress_",)
K4 = ("hypotheses_kernel",)
MODES = ("uniform", "adaptive")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def run(model, inputs, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        for _ in range(iters):
            model(*inputs)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters * 1e3


def kernel_ms(model, inputs, iters):
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            model(*inputs)
        torch.cuda.synchronize()
    out = {"K1": 0.0, "K3": 0.0, "K4": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if any(k in e.key for k in K1):
            out["K1"] += t / 1e3 / iters
        elif any(k in e.key for k in K3) and "bwd" not in e.key:
            out["K3"] += t / 1e3 / iters
        elif any(k in e.key for k in K4):
            out["K4"] += t / 1e3 / iters
    return {k: round(v, 4) for k, v in out.items()}


def _stage_planes(model, s):
    """Runs the model with a hook on the hypotheses of stages 1 and 0 -> {l: (B,D,h,w) planes}."""
    from casmvsnet_pl_b200 import ops
    planes = {}
    orig = ops.warp_cost_ladder, ops.warp_cost

    def ladder(feats, pm, lad, *a, **k):
        planes[lad.h] = lad.materialize()
        return orig[0](feats, pm, lad, *a, **k)

    def tensor(feats, pm, dv, *a, **k):
        planes[dv.shape[-2]] = dv
        return orig[1](feats, pm, dv, *a, **k)
    ops.warp_cost_ladder, ops.warp_cost = ladder, tensor
    try:
        out = model(s["imgs"], s["proj_mats"], s["init_depth_min"], s["depth_interval"])
    finally:
        ops.warp_cost_ladder, ops.warp_cost = orig
    return out, planes


def study(steps=128, tilts=(0.0, 2.25)):
    """The inverse study's settings (8 views, 640x512, V = 5, K = 1, adam at lr 1e-3, --seed 0,
    smoothness weight 0.01) for `steps` optimiser steps on a textured capture at each tilt, once per
    mode from the same random initialisation.  Level-0 error in uniform-mode intervals of each
    reference view against the float64 ground truth, and per stage 1 / 0 the coverage of the ground
    truth by the stage's planes and their median spacing."""
    import os
    import tempfile

    from casmvsnet_pl_b200 import synth_scenes, train, train_data
    out = []
    for tilt in tilts:
        with tempfile.TemporaryDirectory() as root:
            cap = os.path.join(root, "capture")
            synth_scenes.make_colmap(cap, n_views=8, image_wh=(640, 512), n_points=3000, seed=5,
                                     textured=True, tilt=tilt)
            ts = train_data.ColmapTrainSet(cap, n_views=5, img_wh=(640, 512), device="cuda",
                                           log=lambda m: None)
            sc = ts.scan.scene
            gts = []
            for ids in ts.ids:
                v = ids[0]
                K = sc.K[v].copy()
                K[0] *= 640 / sc.wh[v, 0]
                K[1] *= 512 / sc.wh[v, 1]
                gts.append(torch.from_numpy(synth_scenes.height_field_depth(K, sc.E[v], (640, 512), 3.0,
                                                                            tilt)[0]).cuda())

            @torch.no_grad()
            def error(model):
                model.eval()
                errs, cov, spacing = [], {1: [], 0: []}, {1: [], 0: []}
                for i, gt in enumerate(gts):
                    s = ts.batch([i])
                    res, planes = _stage_planes(model, s)
                    dint = float(s["depth_interval"])
                    errs.append(((res["depth_0"][0].double() - gt).abs() / dint).reshape(-1))
                    for l, hl in ((1, 256), (0, 512)):
                        p = planes[hl][0].double()
                        g = torch.nn.functional.interpolate(gt[None, None], size=p.shape[-2:],
                                                            mode="nearest")[0, 0]
                        cov[l].append(((g >= p[0]) & (g <= p[-1])).double().reshape(-1))
                        spacing[l].append(((p[-1] - p[0]) / (p.shape[0] - 1) / dint).reshape(-1))
                e = torch.cat(errs)
                res = {"mean_intervals": round(float(e.mean()), 4),
                       **{f"within_{t}": round(float((e <= t).double().mean()), 4) for t in (1, 2, 4)}}
                for l in (1, 0):
                    res[f"coverage_{l}"] = round(float(torch.cat(cov[l]).mean()), 4)
                    res[f"median_spacing_{l}"] = round(float(torch.cat(spacing[l]).median()), 4)
                return res

            argv = ["--dataset_name", "colmap", "--loss_type", "photo", "--root_dir", cap, "--img_wh",
                    "640", "512", "--n_views", "5", "--num_epochs", str(max(1, -(-steps // len(gts)))),
                    "--optimizer", "adam", "--lr", "1e-3", "--seed", "0", "--log_every", "1000",
                    "--num_workers", "0", "--photo_topk", "1", "--smooth_weight", "0.01"]
            here = os.getcwd()
            for mode in MODES:
                a = train.parse_args(argv + ["--depth_sampling", mode])
                torch.manual_seed(0)
                before = error(train.build_model(a, "cuda"))
                os.chdir(root)
                try:
                    trainer = train.main(argv + ["--depth_sampling", mode, "--exp_name", mode])
                finally:
                    os.chdir(here)
                out.append({"mode": mode, "tilt": tilt, "steps": trainer.global_step,
                            "before": before, "after": error(trainer.model)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--study", action="store_true", help="run the synthetic quality study only")
    ap.add_argument("--steps", type=int, default=128)
    a = ap.parse_args()
    gpu = card()
    if a.study:
        for rec in study(a.steps):
            print(json.dumps(dict(study=rec, gpu=gpu)), flush=True)
        return
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN, precision="tf32")
    synth.randomize_model_(model, 0)
    model = model.eval().cuda()
    for name, (W, H, V) in SIZES.items():
        imgs, pm, dmin, dint = synth.make_inputs(B=1, V=V, W=W, H=H, seed=0)
        inputs = (imgs.cuda(), pm.cuda(), dmin, dint)
        times = {m: [] for m in MODES}
        for mode in times:
            model.set_depth_sampling(mode)
            run(model, inputs, 3)
        for _ in range(a.rounds):
            for mode in times:
                model.set_depth_sampling(mode)
                times[mode].append(round(run(model, inputs, a.iters), 4))
        for mode in times:
            model.set_depth_sampling(mode)
            print(json.dumps(dict(size=name, mode=mode, ms_per_map=times[mode],
                                  kernels_ms=kernel_ms(model, inputs, 10), gpu=gpu)), flush=True)


if __name__ == "__main__":
    main()
