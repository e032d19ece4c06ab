"""Per-layer timing of the tf32 CostRegNet stack (casmvs_costreg_fwd) at the three cascade stages
of the flagship configuration (640x512, V=3, D=48/32/8): one JSON line per layer with its time,
algorithmic HBM bytes, achieved GB/s and the multiple of its HBM time at the data-sheet rate.

Each stage runs on a blocked, TF32-rounded cost volume of the shape and layout that
CascadeMVSNet.run_stage hands the stack (random values: the layers' speed does not depend on
them), with a randomly initialised CostRegNet.  One full two-layer-tail call fills the
workspace; then every layer is launched alone (casmvs_costreg_layer_fwd) on those activations,
with the L2 flushed (256 MiB memset) before each timed launch, CUDA events around it, and the
median of --reps runs.  --fused adds the fused conv11 + prob kernel (layer 11) next to the sum of
conv11 and prob.

    python bench_costreg_layers.py [--reps 25] [--fused]
"""
import argparse
import json
import statistics
import subprocess
import sys

import torch

from casmvsnet_pl_b200 import ABN, _lib, ops

HBM_GBPS = 3350.0                     # H100 SXM data sheet; the card's limit is printed beside
STAGES = ((2, 32, 48, 128, 160), (1, 16, 32, 256, 320), (0, 8, 8, 512, 640))   # level, Cin, D, h, w
NAMES = ("conv0", "conv1", "conv2", "conv3", "conv4", "conv5", "conv6", "conv7", "conv9",
         "conv11", "prob", "conv11+prob fused")


def layer_bytes(cin, n):
    """Algorithmic fp32 bytes of each layer (input, skip, output read / written once), n = D*h*w
    voxels of the stage's full-resolution volume."""
    v = 4 * n
    c = [cin * v + 8 * v,                          # conv0: cost volume -> c0
         8 * v + 16 * v / 8,                       # conv1 (stride 2)
         16 * v / 8 * 2,                           # conv2
         16 * v / 8 + 32 * v / 64,                 # conv3 (stride 2)
         32 * v / 64 * 2,                          # conv4
         32 * v / 64 + 64 * v / 512,               # conv5 (stride 2)
         64 * v / 512 * 2,                         # conv6
         64 * v / 512 + 2 * 32 * v / 64,           # conv7 (transposed) + c4 skip
         32 * v / 64 + 2 * 16 * v / 8,             # conv9 + c2 skip
         16 * v / 8 + 2 * 8 * v,                   # conv11 + c0 skip
         8 * v + v,                                # prob -> logits
         16 * v / 8 + 8 * v + v]                   # fused: u9, c0 -> logits
    return c


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--fused", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_costreg_layers.py needs a GPU")
    from casmvsnet_pl_b200.models.mvsnet import CostRegNet
    dev = "cuda:0"
    lib = _lib.load()
    print(json.dumps({"card": card(), "hbm_gbps_datasheet": HBM_GBPS}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    totals = {}
    for level, cin, D, h, w in STAGES:
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
        layers = list(range(11)) + ([11] if args.fused else [])
        nbytes = layer_bytes(cin, D * h * w)
        for i in layers:
            ts = []
            for it in range(3 + args.reps):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _lib.check(lib.casmvs_costreg_layer_fwd(*a, i, ops._stream()), "costreg_layer")
                e1.record()
                torch.cuda.synchronize()
                if it >= 3:
                    ts.append(e0.elapsed_time(e1))
            ms = statistics.median(ts)
            gbps = nbytes[i] / (ms * 1e-3) / 1e9
            totals.setdefault(NAMES[i], 0.0)
            totals[NAMES[i]] += ms
            print(json.dumps({"level": level, "layer": NAMES[i], "ms": round(ms, 5),
                              "bytes": int(nbytes[i]), "GBps": round(gbps, 1),
                              "x_hbm_time": round(HBM_GBPS / gbps, 2)}), flush=True)
        del x, ws, logits
    summary = {"sum_over_stages_ms": {k: round(v, 4) for k, v in totals.items()},
               "stack_ms": round(sum(v for k, v in totals.items() if k != NAMES[11]), 4),
               "conv11+prob_ms": round(totals["conv11"] + totals["prob"], 4)}
    if args.fused:
        summary["fused_ms"] = round(totals[NAMES[11]], 4)
    summary["card"] = card()
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
