"""Training-step measurement at the reference's training shape: 640x512, V = 3, D = 48/32/8,
on a full-size synthetic DTU training scan (synth_scenes.make_dtu_train) written to a
temporary directory.

    python bench_train.py [--steps 50] [--warmup 5] [--out result.json]
    python bench_train.py --profile [--out profile.json]      # one step under torch.profiler

Default run, one JSON object: the card's name and power limit; the host data time per sample
(decode + slice in the main process); for fp32 and tf32 at B = 1 and 2 the step time (forward,
SL1 loss, backward, SGD step, each step ended by a device synchronise), median and mean over
--steps steps after --warmup, and the peak allocated / reserved memory of the step.
--profile: the kernels of one fp32 B = 1 step (and one B = 2 step) grouped into families, with
each family's share of the step's kernel time and the top kernels by time.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from casmvsnet_pl_b200 import train, train_data  # noqa: E402
from casmvsnet_pl_b200.synth_scenes import make_dtu_train  # noqa: E402

FAMILIES = [  # (family, substrings of kernel names), first match wins
    ("conv3d_wgrad", ("conv3d_wgrad",)),
    ("conv3d fwd/dgrad (own)", ("conv3d", "costreg", "tma_conv", "direct_conv")),
    ("warp_cost fwd/bwd (own)", ("warp_cost", "homo_warp")),
    ("regress fwd/bwd (own)", ("regress", "hypotheses", "depth_first")),
    ("sl1 loss (own)", ("sl1_",)),
    ("FeatureNet cuDNN conv", ("cudnn", "xmma", "implicit", "conv2d", "wgrad", "dgrad", "sm90_", "cutlass",
                               "gemm", "fft", "winograd")),
    ("batch norm", ("batch_norm", "bn_", "welford")),
    ("optimizer", ("multi_tensor", "foreach", "sgd", "adam")),
]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else \
        torch.cuda.get_device_name(0)


def family(name):
    n = name.lower()
    for fam, keys in FAMILIES:
        if any(k in n for k in keys):
            return fam
    return "elementwise / other"


def batches(ds, B, n):
    """n distinct device batches of B samples (uploaded once, reused in turn)."""
    out = []
    for j in range(n):
        idx = [(j * B + k) % len(ds) for k in range(B)]
        out.append(train_data.to_device(torch.utils.data.default_collate([ds[i] for i in idx]), "cuda:0"))
    return out


def make_trainer(precision):
    a = train.build_parser().parse_args(["--precision", precision, "--optimizer", "sgd"])
    torch.manual_seed(0)
    return train.Trainer(a, train.build_model(a, "cuda:0"), "cuda:0")


def time_steps(tr, bs, warmup, steps):
    for i in range(warmup):
        tr.train_step(bs[i % len(bs)])
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for i in range(steps):
        t0 = time.perf_counter()
        tr.train_step(bs[i % len(bs)])
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return {"median_ms": 1e3 * statistics.median(times), "mean_ms": 1e3 * statistics.mean(times),
            "min_ms": 1e3 * min(times), "max_ms": 1e3 * max(times), "steps": steps,
            "peak_allocated_GB": torch.cuda.max_memory_allocated() / 1e9,
            "peak_reserved_GB": torch.cuda.max_memory_reserved() / 1e9}


def profile_step(tr, bs):
    from torch.profiler import ProfilerActivity, profile
    for b in bs:
        tr.train_step(b)                      # warm
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        tr.train_step(bs[0])
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            k = kern.setdefault(e.name, [0.0, 0])
            k[0] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            k[1] += 1
    total = sum(v[0] for v in kern.values())
    fams = {}
    for n, (t, _) in kern.items():
        fams[family(n)] = fams.get(family(n), 0.0) + t
    top = sorted(kern.items(), key=lambda kv: -kv[1][0])[:25]
    return {"kernel_time_ms": total / 1e3,
            "families": {f: {"ms": t / 1e3, "share": t / total} for f, t in
                         sorted(fams.items(), key=lambda kv: -kv[1])},
            "top_kernels": [{"name": n[:120], "ms": t / 1e3, "calls": c, "family": family(n)}
                            for n, (t, c) in top]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train.py measures on a CUDA GPU")
    res = {"card": card(), "shape": "640x512, V=3, D=48/32/8"}
    with tempfile.TemporaryDirectory() as tmp:
        root = make_dtu_train(os.path.join(tmp, "dtu"), seed=0)
        ds = train_data.DTUTrainDataset(root, ["scan1"])
        if a.profile:
            for B in (1, 2):
                tr = make_trainer("fp32")
                res[f"fp32_B{B}"] = profile_step(tr, batches(ds, B, 2))
                del tr
                torch.cuda.empty_cache()
        else:
            t0 = time.perf_counter()
            n = 14
            for i in range(n):
                ds[i]
            res["host_data_ms_per_sample"] = 1e3 * (time.perf_counter() - t0) / n
            for prec in ("fp32", "tf32"):
                for B in (1, 2):
                    tr = make_trainer(prec)
                    res[f"{prec}_B{B}"] = time_steps(tr, batches(ds, B, 4), a.warmup, a.steps)
                    del tr
                    torch.cuda.empty_cache()
                    print(prec, B, res[f"{prec}_B{B}"], file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
