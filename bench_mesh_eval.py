"""Time mesh scoring on the GPU (mesh_sample.py, dtu_eval.evaluate_mesh, tnt_eval.evaluate_mesh)
on meshes of the sizes a user scores:

- a DTU-sized synth_dtu scene (3 M STL points, about 346 mm across), its height field
  triangulated at 0.4 mm (about 1.5 M faces), then decimated to 10 % and 1 % (simplify.py), each
  scored at the 0.2 mm thinning distance;
- the synth_tnt.make_scene surfaces triangulated in the ground-truth frame to about 2 M faces,
  scored at tau / 4.

Per mesh: the points kernel alone (CUDA events, median of --repeats launches after a warm-up,
with the bytes it writes over that time against the data sheet's 3.35 TB/s), sample_surface end
to end, every evaluate_mesh phase from its time_s, and the peak allocation of evaluate_mesh over
the mesh's resident size, also per sample (what mesh_sample.BYTES_PER_SAMPLE budgets).  Prints
one JSON line per mesh with the card name and power limit read in the same run.

    python bench_mesh_eval.py [--n_stl 3000000] [--step 0.4] [--ratios 0.1 0.01] [--tnt_res 4.8]
"""
import argparse
import json
import statistics
import tempfile

import numpy as np
import torch

from bench_mesh import card
from casmvsnet_pl_b200 import dtu_eval, mesh_sample, simplify, synth_dtu, synth_tnt, tnt_eval

HBM_BYTES_PER_S = 3.35e12


def kernel_ms(v, f, spacing, repeats):
    n, count, start = mesh_sample.sample_counts(v, f, spacing)
    S = int(count.sum())
    mesh_sample.sample_points(v, f, n, start, S)                     # warm-up
    times = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = mesh_sample.sample_points(v, f, n, start, S)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
        del out
    return statistics.median(times), S


def sample_ms(v, f, spacing, repeats):
    mesh_sample.sample_surface(v, f, spacing)
    times = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = mesh_sample.sample_surface(v, f, spacing)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
        del out
    return statistics.median(times)


def bench(label, v, f, spacing, score, repeats, name, power):
    v = torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda()
    f = torch.from_numpy(np.ascontiguousarray(f, np.int32)).cuda()
    k_ms, S = kernel_ms(v, f, spacing, repeats)
    s_ms = sample_ms(v, f, spacing, repeats)
    score(v, f)                                                       # warm-up
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    r = score(v, f)
    peak = torch.cuda.max_memory_allocated() - base
    phases = {k: round(x, 4) for k, x in r["time_s"].items() if k.endswith("_s")}
    print(json.dumps(dict(mesh=label, faces=len(f), spacing=spacing, samples=S,
                          points_kernel_ms=round(k_ms, 3),
                          points_kernel_tb_per_s=round(12 * S / (k_ms * 1e-3) / 1e12, 3),
                          points_kernel_share_of_hbm=round(12 * S / (k_ms * 1e-3) / HBM_BYTES_PER_S, 3),
                          sample_surface_ms=round(s_ms, 3), evaluate_s=phases,
                          peak_bytes=peak, peak_bytes_per_sample=round(peak / S, 1),
                          gpu=name, power_limit=power)), flush=True)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--n_stl", type=int, default=3_000_000)
    ap.add_argument("--step", type=float, default=0.4)
    ap.add_argument("--ratios", nargs="*", type=float, default=[0.1, 0.01])
    ap.add_argument("--tnt_res", type=float, default=4.8)
    ap.add_argument("--repeats", type=int, default=20)
    a = ap.parse_args(argv)
    name, power = card()
    with tempfile.TemporaryDirectory() as tmp:
        synth_dtu.make_scene(tmp, 1, n_stl=a.n_stl, n_data=1000, seed=0)
        stl = dtu_eval.read_points(dtu_eval.stl_path(tmp, 1))
        v, f, _, _ = synth_dtu.height_mesh(stl, a.step)

        def dtu(v, f):
            return dtu_eval.evaluate_mesh((v, f), 1, tmp)
        bench(f"dtu_height_{a.step}mm", v, f, dtu_eval.DST, dtu, a.repeats, name, power)
        for ratio in a.ratios:
            V, _, F, _ = simplify.simplify_mesh(
                torch.from_numpy(v).cuda(), torch.zeros(len(v), 3, dtype=torch.uint8, device="cuda"),
                torch.from_numpy(f).cuda(), max(1, round(ratio * len(f))), log=lambda *_: None)
            bench(f"dtu_height_{a.step}mm_{ratio:g}", V.cpu().numpy(), F.cpu().numpy(), dtu_eval.DST,
                  dtu, a.repeats, name, power)
    with tempfile.TemporaryDirectory() as tmp:
        sc = synth_tnt.make_scene(tmp, n_gt=2_000_000, n_rec=1000, seed=0)
        P, f = synth_tnt.surface_mesh(a.tnt_res)
        T = np.linalg.inv(sc["rec_to_gt"])
        v = (P @ T[:3, :3].T + T[:3, 3]).astype(np.float32)

        def tnt(v, f):
            return tnt_eval.evaluate_mesh((v, f), sc["run_dir"], sc["gt_dir"], sc["scene"],
                                          tau=sc["tau"], images=sc["images"])
        bench(f"tnt_surfaces_res{a.tnt_res:g}", v, f, sc["tau"] / 4, tnt, a.repeats, name, power)


if __name__ == "__main__":
    main()
