"""Timing of the training panel strip (csrc/visual.cu, visual.training_panel) against the
original project's host chain, at 640x512 (DTU), 768x576 (BlendedMVS) and 1152x864:

  panel    training_panel on device inputs (the min/max pass and the drawing pass) back to back:
           per call, the larger of the two kernels and the host side of a call.  CUDA events
           around --calls back-to-back calls, per call; median of --reps windows after --warmup.
  kernels  device time of the two kernels per call, from torch.profiler with CUDA activities
           over --calls calls, in a pass of its own.
  logged   what the trainer spends per logged image: training_panel and its one device -> host
           copy of the (H, 4W, 3) uint8 strip; host clock to the end of the copy, median.
  host     the original's path on the same device tensors: Normalize on the device and .cpu(),
           then per depth / confidence panel .cpu(), numpy (nan_to_num, min / max, scale, cast),
           cv2.applyColorMap, PIL Image.fromarray, ToTensor; torch.stack and TensorBoard's
           conversion of the stack to the uint8 strip.  Host clock, median.

Each size also checks that the host chain's strip equals the kernel's, byte for byte.  Prints the
card's name and power limit, then one JSON line per size.  Writes nothing.

    python bench_visual.py [--reps 9] [--warmup 3] [--calls 50]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_view_select import card  # noqa: E402
from casmvsnet_pl_b200 import visual  # noqa: E402

SIZES = {"dtu_640x512": (512, 640), "blendedmvs_768x576": (576, 768), "1152x864": (864, 1152)}
DEV = "cuda:0"


def inputs(H, W, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    img = torch.randn(3, H, W, generator=g, device=DEV)
    mask = torch.rand(H, W, generator=g, device=DEV) > 0.2
    gt = (425.0 + 510.0 * torch.rand(H, W, generator=g, device=DEV)) * mask
    pred = gt + 20.0 * torch.randn(H, W, generator=g, device=DEV)
    conf = torch.rand(H, W, generator=g, device=DEV)
    return img, gt, pred, conf, mask


def host_chain(img, gt, pred, conf, mask):
    """The original's logging path for one stack, from device tensors to the uint8 strip."""
    import cv2
    import torchvision.transforms as T
    from PIL import Image
    from torch.utils.tensorboard._utils import convert_to_HWC

    def coloured(grey, cmap):
        return T.ToTensor()(Image.fromarray(cv2.applyColorMap(grey, cmap)))

    def depth_panel(d):
        x = np.nan_to_num(d.cpu().numpy())
        lo, hi = np.min(x[x > 0]), np.max(x)
        return coloured((255 * ((x - lo) / (hi - lo + 1e-8))).astype(np.uint8), cv2.COLORMAP_JET)

    unnorm = T.Normalize(mean=[-0.485 / 0.229, -0.456 / 0.224, -0.406 / 0.225],
                         std=[1 / 0.229, 1 / 0.224, 1 / 0.225])
    stack = torch.stack([unnorm(img).cpu(), depth_panel(gt), depth_panel(pred * mask),
                         coloured((255 * (conf * mask)).cpu().numpy().astype(np.uint8),
                                  cv2.COLORMAP_BONE)])
    hwc = convert_to_HWC(stack.numpy(), "NCHW").astype(np.float32)
    return (hwc * 255).clip(0, 255).astype(np.uint8)


def time_kernel(args, reps, warmup, calls):
    for _ in range(warmup):
        visual.training_panel(*args)
    torch.cuda.synchronize()
    per_call = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            visual.training_panel(*args)
        e1.record()
        e1.synchronize()
        per_call.append(e0.elapsed_time(e1) / calls)
    return statistics.median(per_call)


def kernel_us(args, calls):
    """Mean device time per call of each of the two kernels, in microseconds."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            visual.training_panel(*args)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.key.startswith("casmvs::") or "visual_" in e.key:
            name = "minmax" if "minmax" in e.key else "draw" if "draw" in e.key else e.key
            out[name] = round(e.device_time_total / calls, 2)
    return out


def time_host(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--calls", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_visual.py needs a CUDA GPU")
    name, power = card()
    print(f"card: {name}, power limit {power}")
    for case, (H, W) in SIZES.items():
        args = inputs(H, W, H + W)
        same = np.array_equal(host_chain(*args), visual.training_panel(*args).cpu().numpy())
        res = {"metric": "visual_panel", "case": case, "H": H, "W": W,
               "panel_ms": round(time_kernel(args, a.reps, a.warmup, a.calls), 4),
               "kernels_us": kernel_us(args, a.calls),
               "logged_ms": round(time_host(lambda: visual.training_panel(*args).cpu(),
                                            a.reps, a.warmup), 4),
               "host_chain_ms": round(time_host(lambda: host_chain(*args), a.reps, a.warmup), 3),
               "strips_equal": bool(same), "card": name, "power_limit": power}
        print(json.dumps(res), flush=True)
        if not same:
            raise SystemExit(f"{case}: the kernel's strip differs from the host chain's")


if __name__ == "__main__":
    main()
