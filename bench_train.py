"""Training-step measurement at the reference's training shape: 640x512, V = 3, D = 48/32/8,
on a full-size synthetic DTU training scan (synth_scenes.make_dtu_train) written to a
temporary directory.

    python bench_train.py [--steps 50] [--warmup 5] [--out result.json]
    python bench_train.py --profile [--out profile.json]      # one step under torch.profiler
    python bench_train.py --dataset blendedmvs [--steps 50] [--warmup 5]
    python bench_train.py --deterministic [--dataset blendedmvs] [--steps 50] [--warmup 5]

Default run, one JSON object: the card's name and power limit; the host data time per sample
(decode + slice in the main process); for fp32 and tf32 at B = 1 and 2 the step time (forward,
SL1 loss, backward, SGD step, each step ended by a device synchronise), median and mean over
--steps steps after --warmup, and the peak allocated / reserved memory of the step.
--profile: the kernels of one fp32 B = 1 step (and one B = 2 step) grouped into families, with
each family's share of the step's kernel time and the top kernels by time.
--dataset blendedmvs: the same at BlendedMVS's training shape, 768x576, on two synthetic
dataset_low_res scans with native-size JPEGs (synth_scenes.make_blendedmvs_train), training
split (colour-jittered batches); the host data time is the decode-only worker's, and the
object adds the time of the same jitter done with Pillow on the host (ImageEnhance, what
torchvision's ColorJitter calls) and of the fused device kernel (CUDA events).
--deterministic: the same steps under torch.use_deterministic_algorithms(True), as
train.py --deterministic runs them (deterministic backward kernels, no cuDNN autotuning); the
object says so in "deterministic".
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
from casmvsnet_pl_b200.synth_scenes import make_blendedmvs_train, make_dtu_train  # noqa: E402

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


def host_pil_jitter_ms(ds, n):
    """Per sample: Pillow's brightness and contrast enhancers on the sample's V decoded views,
    in each view's drawn order (host work the device kernel replaces)."""
    from PIL import Image, ImageEnhance
    samples = [ds[i % len(ds)] for i in range(n)]
    ims = [[Image.fromarray(v) for v in s["imgs_u8"].numpy()] for s in samples]
    t0 = time.perf_counter()
    for s, views in zip(samples, ims):
        for im, (bf, b, c) in zip(views, s["jitter"].tolist()):
            for fn in ("b", "c") if bf else ("c", "b"):
                im = ImageEnhance.Brightness(im).enhance(b) if fn == "b" else \
                    ImageEnhance.Contrast(im).enhance(c)
    return 1e3 * (time.perf_counter() - t0) / n


def jitter_kernel_ms(ds, B, iters=200):
    """CUDA-event time of io.jitter_normalize_images on the B * V images of a batch."""
    from casmvsnet_pl_b200 import io
    batch = torch.utils.data.default_collate([ds[i] for i in range(B)])
    _, V, H, W, _ = batch["imgs_u8"].shape
    u8 = batch["imgs_u8"].reshape(B * V, H, W, 3).cuda()
    jit = batch["jitter"].reshape(B * V, 3).cuda()
    out = torch.empty(B * V, 3, H, W, device="cuda")
    for _ in range(10):
        io.jitter_normalize_images(u8, jit, out=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        io.jitter_normalize_images(u8, jit, out=out)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_blendedmvs(a, tmp):
    res = {"card": card(), "dataset": "blendedmvs", "shape": "768x576, V=3, D=48/32/8"}
    root = make_blendedmvs_train(os.path.join(tmp, "blendedmvs"), n_views=(8, 6), image_wh=(768, 576))
    ds = train_data.BlendedMVSTrainDataset(root, "train")
    n = len(ds)
    t0 = time.perf_counter()
    for i in range(n):
        ds[i]
    res["host_data_ms_per_sample"] = 1e3 * (time.perf_counter() - t0) / n
    res["host_pil_jitter_ms_per_sample"] = host_pil_jitter_ms(ds, n)
    for B in (1, 2):
        res[f"jitter_kernel_ms_B{B}"] = jitter_kernel_ms(ds, B)
    for prec in ("fp32", "tf32"):
        for B in (1, 2):
            tr = make_trainer(prec)
            res[f"{prec}_B{B}"] = time_steps(tr, batches(ds, B, 3), a.warmup, a.steps)
            del tr
            torch.cuda.empty_cache()
            print(prec, B, res[f"{prec}_B{B}"], file=sys.stderr, flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dataset", default="dtu", choices=["dtu", "blendedmvs"],
                    help="training shape and data: DTU 640x512 (default) or BlendedMVS 768x576")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--deterministic", action="store_true",
                    help="time the steps with deterministic algorithms on (train.py --deterministic)")
    a = ap.parse_args()
    if a.deterministic:
        train.set_deterministic()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train.py measures on a CUDA GPU")
    if a.dataset == "blendedmvs" and a.profile:
        raise SystemExit("--profile measures the DTU shape only")
    res = {"card": card(), "shape": "640x512, V=3, D=48/32/8", "deterministic": a.deterministic}
    with tempfile.TemporaryDirectory() as tmp:
        if a.dataset == "blendedmvs":
            res = bench_blendedmvs(a, tmp)
            res["deterministic"] = a.deterministic
        else:
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
