"""Time Tanks and Temples scoring (casmvsnet_pl_b200/tnt_eval.py) on a synthetic training scene at
assumed real sizes.

The sizes are assumptions, not measurements of the official data: 20 M ground-truth points and
30 M reconstructed points (a fused cloud of a training scene is tens of millions of points), with
tau = 0.01 (Barn's) on the synth_tnt surfaces, about 37 m^2.  Prints the card name and power limit
read in the same run, the per-phase times (each ends in a device synchronise) and one JSON line.

The float64 restatement (oracle/tnt_eval_oracle.py) is timed on the host on the same generator at
--oracle_points reconstructed points (default 300 k, scaled ground truth); at full size it would
take hours and is not run.

    python bench_tnt_eval.py [--gt_points 20000000] [--rec_points 30000000] [--repeat 2]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--gt_points", type=int, default=20_000_000)
    ap.add_argument("--rec_points", type=int, default=30_000_000)
    ap.add_argument("--tau", type=float, default=0.01)
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--oracle_points", type=int, default=300_000)
    a = ap.parse_args(argv)
    import numpy as np
    import torch

    from casmvsnet_pl_b200 import synth_tnt
    from casmvsnet_pl_b200 import tnt_eval as E
    from oracle import tnt_eval_oracle as O

    if not torch.cuda.is_available():
        raise SystemExit("bench_tnt_eval needs a GPU")
    print(f"card: {card()}", flush=True)
    with tempfile.TemporaryDirectory() as d:
        t = time.perf_counter()
        s = synth_tnt.make_scene(d, n_gt=a.gt_points, n_rec=a.rec_points, tau=a.tau, seed=0)
        print(f"scene: {a.gt_points} ground-truth and {a.rec_points} reconstructed points written "
              f"in {time.perf_counter() - t:.1f} s", flush=True)
        pts = torch.from_numpy(E.read_points(s["ply"])).cuda()
        runs = []
        for k in range(a.repeat + 1):           # the first run warms up kernels and allocator
            r = E.evaluate_scene(pts, s["run_dir"], s["gt_dir"], s["scene"], tau=a.tau,
                                 images=s["images"])
            if k:
                runs.append(r)
        r = runs[-1]
        ph = {k: min(x["time_s"][k] for x in runs) for k in r["time_s"]}
        print("counts:", json.dumps(r["counts"]))
        print("stages:", [(st["iterations"], round(st["fitness"], 4), round(st["rmse"], 6))
                          for st in r["stages"]])
        print(f"F {r['fscore']:.4f}  P {r['precision']:.4f}  R {r['recall']:.4f}")
        print("GPU phases (s, best of %d): " % len(runs) + "  ".join(f"{k[:-2]} {v:.3f}"
                                                                     for k, v in ph.items()))
        gpu_total = ph["total_s"] - ph["load_s"]
        # the restatement, on the host, at a reduced size
        frac = a.oracle_points / a.rec_points
        so = synth_tnt.make_scene(os.path.join(d, "small"), n_gt=int(a.gt_points * frac),
                                  n_rec=a.oracle_points, tau=a.tau, seed=0)
        ro = E.evaluate_scene(so["ply"], so["run_dir"], so["gt_dir"], so["scene"], tau=a.tau,
                              images=so["images"])
        rec = E.read_points(so["ply"])
        gt = E.read_points(os.path.join(so["gt_dir"], so["scene"], f"{so['scene']}.ply"))
        vol = E.read_crop(os.path.join(so["gt_dir"], so["scene"], f"{so['scene']}.json"))
        t = time.perf_counter()
        want = O.evaluate(rec, gt, np.array(ro["alignment"]["T0"]), vol, a.tau)
        oracle_s = time.perf_counter() - t
        small_gpu = ro["time_s"]["total_s"] - ro["time_s"]["load_s"] - ro["time_s"]["align_s"]
        print(f"oracle (host, float64) at {a.oracle_points} reconstructed points: {oracle_s:.1f} s "
              f"(GPU at that size: {small_gpu:.3f} s); F {want['fscore']:.4f} vs GPU {ro['fscore']:.4f}")
    print(json.dumps(dict(metric="tnt_eval_s", value=round(gpu_total, 4), unit="s", card=card(),
                          gt_points=a.gt_points, rec_points=a.rec_points, tau=a.tau,
                          phases_s={k: round(v, 4) for k, v in ph.items()},
                          oracle_points=a.oracle_points, oracle_s=round(oracle_s, 2),
                          gpu_at_oracle_size_s=round(small_gpu, 4))))


if __name__ == "__main__":
    main()
