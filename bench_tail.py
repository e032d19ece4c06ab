"""Timing of CostRegNet's fused conv11 + prob tail (conv3d_tail.cu, casmvs_costreg_layer_fwd
layer 11) alone, at the three cascade stages of the flagship configuration (640x512, V=3,
D=48/32/8) and at the full-resolution stage of 1152x864 and 1920x1056 (D=8): one JSON line per
stage with its time, algorithmic HBM bytes (u9 and c0 read, logits written, once) and the
multiple of its HBM time at the data-sheet rate.

Same set-up as bench_costreg_layers.py: a blocked, TF32-rounded input and a randomly initialised
CostRegNet; one full stack call fills the workspace; then the tail is launched alone with the L2
flushed (256 MiB memset) before each launch, CUDA events around it, and the median of --reps.

    python bench_tail.py [--reps 25]
"""
import argparse
import json
import statistics
import sys

import torch

from bench_costreg_layers import HBM_GBPS, card
from casmvsnet_pl_b200 import ABN, _lib, ops

STAGES = (("640x512", 2, 32, 48, 128, 160), ("640x512", 1, 16, 32, 256, 320),
          ("640x512", 0, 8, 8, 512, 640), ("1152x864", 0, 8, 8, 864, 1152),
          ("1920x1056", 0, 8, 8, 1056, 1920))          # config, level, Cin, D, h, w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=25)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tail.py needs a GPU")
    from casmvsnet_pl_b200.models.mvsnet import CostRegNet
    dev = "cuda:0"
    lib = _lib.load()
    print(json.dumps({"card": card(), "hbm_gbps_datasheet": HBM_GBPS}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    total = 0.0
    for cfg, level, cin, D, h, w in STAGES:
        torch.manual_seed(level)
        net = CostRegNet(cin, ABN)
        with torch.no_grad():
            for m in net.modules():
                if hasattr(m, "running_mean"):
                    m.weight.uniform_(0.5, 1.5)
                    m.bias.normal_(0.0, 0.1)
        params = net.eval().to(dev).requires_grad_(False).packed_params()
        x = torch.randn(1, cin // 4, D, h, w, 4, device=dev)
        x = ((x.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
        ws_bytes = lib.casmvs_costreg_workspace_bytes(1, cin, D, h, w)
        ws = torch.empty(ws_bytes // 4, device=dev)
        logits = torch.empty(1, D, h, w, device=dev)
        prec = ops.TF32 | ops.BLOCKED
        a = (ops._ptr(x), ops._ptr(params), ops._ptr(logits), 1, cin, D, h, w, prec,
             ops._ptr(ws), ws_bytes)
        _lib.check(lib.casmvs_costreg_fwd(*a, ops._stream()), "costreg")
        ts = []
        for it in range(3 + args.reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(lib.casmvs_costreg_layer_fwd(*a, 11, ops._stream()), "costreg_layer")
            e1.record()
            torch.cuda.synchronize()
            if it >= 3:
                ts.append(e0.elapsed_time(e1))
        ms = statistics.median(ts)
        v = 4 * D * h * w
        nbytes = 16 * v / 8 + 8 * v + v                 # u9, c0 -> logits
        gbps = nbytes / (ms * 1e-3) / 1e9
        if cfg == "640x512":
            total += ms
        print(json.dumps({"config": cfg, "level": level, "ms": round(ms, 5),
                          "min_ms": round(min(ts), 5), "max_ms": round(max(ts), 5),
                          "bytes": int(nbytes), "GBps": round(gbps, 1),
                          "x_hbm_time": round(HBM_GBPS / gbps, 2)}), flush=True)
        del x, ws, logits
    print(json.dumps({"640x512_sum_ms": round(total, 4), "card": card()}), flush=True)


if __name__ == "__main__":
    main()
