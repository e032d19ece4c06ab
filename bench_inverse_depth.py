"""Inverse-depth plane sweep (README "Wide depth ranges"): cascade time per depth map, uniform
against inverse sampling, alternating in one process, at cfg2 (640x512, V = 3) and 1152x864
(V = 5), and per-kernel K1 / K3 device times from torch.profiler.  K1 may halve its depth runs
more often in the inverse mode (near planes move pixels further); the profiler rows show whether
it costs time.  Prints one JSON line per row, with the card name and power limit read in the same
run.

--study fine-tunes the network with the photometric loss on a synthetic capture whose depths
span a ratio of about 10-15 in each view (synth_scenes.make_colmap(tilt=2.25)), once per sampling mode
from the same seed, and reports the relative depth error against the float64 ground truth over
the nearest and the farthest third of the depths.

    python bench_inverse_depth.py [--iters 30] [--rounds 3]
    python bench_inverse_depth.py --study [--epochs 16]
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
    out = {"K1": 0.0, "K3": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if any(k in e.key for k in K1):
            out["K1"] += t / 1e3 / iters
        elif any(k in e.key for k in K3) and "bwd" not in e.key:
            out["K3"] += t / 1e3 / iters
    return {k: round(v, 4) for k, v in out.items()}


def study(epochs=16, tilt=2.25):
    """bench_photo_loss.study's settings (8 views, 640x512, V = 5, K = 1, adam at lr 1e-3,
    --seed 0, the default smoothness weight) on a tilted textured capture, once per mode.  Before
    and after: the level-0 depth of every reference view in eval mode against the float64 ground
    truth, as |d - gt| / gt: its mean and the share within 0.5 %, 1 % and 2 %, over all pixels and
    over the nearest and the farthest third of the ground-truth depths (pooled over the views)."""
    import os
    import tempfile

    from casmvsnet_pl_b200 import synth_scenes, train, train_data
    out = []
    with tempfile.TemporaryDirectory() as root:
        cap = os.path.join(root, "capture")
        synth_scenes.make_colmap(cap, n_views=8, image_wh=(640, 512), n_points=3000, seed=5,
                                 textured=True, tilt=tilt)
        ts = train_data.ColmapTrainSet(cap, n_views=5, img_wh=(640, 512), device="cuda", log=lambda m: None)
        sc = ts.scan.scene
        gts = []
        for ids in ts.ids:
            v = ids[0]
            K = sc.K[v].copy()
            K[0] *= 640 / sc.wh[v, 0]
            K[1] *= 512 / sc.wh[v, 1]
            gts.append(torch.from_numpy(synth_scenes.height_field_depth(K, sc.E[v], (640, 512), 3.0,
                                                                        tilt)[0]).cuda())
        allgt = torch.cat([g.reshape(-1) for g in gts])
        q1, q2 = (float(x) for x in torch.quantile(allgt[::7].float(), torch.tensor([1 / 3, 2 / 3],
                                                                                    device="cuda")))
        ranges = [(float(ts.batch([i])["init_depth_min"]), float(ts.batch([i])["depth_interval"]))
                  for i in range(len(gts))]

        @torch.no_grad()
        def error(model):
            model.eval()
            rel = []
            for i, gt in enumerate(gts):
                s = ts.batch([i])
                d = model(s["imgs"], s["proj_mats"], s["init_depth_min"], s["depth_interval"])["depth_0"][0]
                rel.append(((d.double() - gt).abs() / gt).reshape(-1))
            rel = torch.cat(rel)
            res = {}
            for name, m in (("all", torch.ones_like(allgt, dtype=torch.bool)), ("near_third", allgt <= q1),
                            ("far_third", allgt > q2)):
                r = rel[m]
                res[name] = {"mean": round(float(r.mean()), 5),
                             **{f"within_{t}%": round(float((r <= t / 100).double().mean()), 4)
                                for t in (0.5, 1, 2)}}
            return res

        argv = ["--dataset_name", "colmap", "--loss_type", "photo", "--root_dir", cap, "--img_wh", "640",
                "512", "--n_views", "5", "--num_epochs", str(epochs), "--optimizer", "adam", "--lr", "1e-3",
                "--seed", "0", "--log_every", "1000", "--num_workers", "0"]
        here = os.getcwd()
        for mode in ("uniform", "inverse"):
            a = train.parse_args(argv + ["--depth_sampling", mode])
            torch.manual_seed(0)
            before = error(train.build_model(a, "cuda"))
            os.chdir(root)
            try:
                trainer = train.main(argv + ["--depth_sampling", mode, "--exp_name", mode])
            finally:
                os.chdir(here)
            out.append({"mode": mode, "tilt": tilt, "gt_depth_min": round(float(allgt.min()), 3),
                        "gt_depth_max": round(float(allgt.max()), 3), "near_third_max": round(q1, 3),
                        "far_third_min": round(q2, 3), "depth_ranges": ranges[:2],
                        "steps": trainer.global_step, "before": before, "after": error(trainer.model)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--study", action="store_true", help="run the synthetic quality study only")
    ap.add_argument("--epochs", type=int, default=16)
    a = ap.parse_args()
    gpu = card()
    if a.study:
        for rec in study(a.epochs):
            print(json.dumps(dict(study=rec, gpu=gpu)), flush=True)
        return
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN, precision="tf32")
    synth.randomize_model_(model, 0)
    model = model.eval().cuda()
    for name, (W, H, V) in SIZES.items():
        imgs, pm, dmin, dint = synth.make_inputs(B=1, V=V, W=W, H=H, seed=0)
        inputs = (imgs.cuda(), pm.cuda(), dmin, dint)
        times = {"uniform": [], "inverse": []}
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
