"""Time the fusion kernel for both consistency rules (fusion.py, csrc/fusion.cu) and compare what
the rules keep on synthetic scenes.

1. One reference view, rule "reference" and rule "dynamic", at 1152x864 and 1920x1056 with 10
   sources: the kernel's device time (torch.profiler), median of --repeats after a warm-up,
   the time of the whole refine_ref_view call (CUDA events), and the bytes per pixel
   csrc/fusion.cu's header counts (4 + S x 4 taps x 16 B read, 4 + 12 + 4 + 12 +
   1 B written) over that time, against the H100 SXM's 3.35 TB/s.
2. fusion.fuse_scan over a 150-view 1152x864 scan (sphere_scene, each view's 10 nearest cameras
   as sources), both rules, median of 3.
3. Quality study (synthetic): sphere_scene's exact depth maps at 1152x864, each view's 10 nearest
   cameras as sources, corrupted with seeded multiplicative noise (sigma 0.2 % of depth) and, on
   2 % of the pixels, 8x8 patches scaled by U(0.8, 1.2); confidence 1, so the geometric check
   alone decides.  Per rule: kept points, the share of kept points within tau of the analytic
   surface (accuracy), and the share of the views' exact surface samples (every pixel that sees
   the surface in some view) within tau of a kept point (completeness, dtu_eval.capped_nn).
   Repeated with the views thinned, so that much of the surface is seen by 2-4 sources only.
Prints one JSON line per row with the card name and power limit read in the same run.

    python bench_fusion.py [--repeats 20] [--scan_views 150]
"""
import argparse
import json
import statistics

import numpy as np
import torch

from bench_mesh import card
from casmvsnet_pl_b200 import dtu_eval, fusion, synth_scenes

HBM_BPS = 3.35e12
RADIUS = 150.0


def bytes_per_pixel(S):
    return 4 + S * 4 * 16 + (4 + 12 + 4 + 12 + 1)


def nearest(views, S):
    C = np.stack([-np.linalg.solve(v["P"][:3, :3].astype(np.float64), v["P"][:3, 3]) for v in views])
    return [[int(j) for j in np.argsort(np.linalg.norm(C - C[i], axis=1))[1:S + 1]] for i in range(len(views))]


def corrupt(depth, gen, sigma=0.002, share=0.02, patch=8):
    """Multiplicative noise, then share of the pixels in patch x patch blocks scaled by U(0.8, 1.2)."""
    H, W = depth.shape
    d = depth * (1 + sigma * torch.randn(H, W, generator=gen, device=depth.device))
    nb = int(share * H * W / patch ** 2)
    ys = torch.randint(0, H - patch, (nb,), generator=gen, device=depth.device)
    xs = torch.randint(0, W - patch, (nb,), generator=gen, device=depth.device)
    sc = 0.8 + 0.4 * torch.rand(nb, generator=gen, device=depth.device)
    for i in range(nb):
        d[ys[i]:ys[i] + patch, xs[i]:xs[i] + patch] *= sc[i]
    return d


def scan_inputs(views, S, seed, device):
    gen = torch.Generator(device=device).manual_seed(seed)
    n = len(views)
    src = nearest(views, S)
    H, W = views[0]["depth"].shape
    depths = {i: corrupt(views[i]["depth"].to(device), gen) for i in range(n)}
    images = {i: views[i]["image"].to(device) for i in range(n)}
    probas = {i: torch.ones(H // 4, W // 4, device=device) for i in range(n)}
    proj = {i: views[i]["P"] for i in range(n)}
    metas = [(i, src[i]) for i in range(n)]
    return metas, depths, probas, images, proj


def time_view(rule, W, H, S, repeats, device):
    views = synth_scenes.sphere_scene(S + 1, (W, H), seed=1, radius=RADIUS, device=device)
    gen = torch.Generator(device=device).manual_seed(1)
    d = [corrupt(v["depth"], gen) for v in views]
    img = [v["image"] for v in views]
    proba = torch.ones(H // 4, W // 4, device=device)
    args = (d[0], views[0]["P"], d[1:], [v["P"] for v in views[1:]], img[0], img[1:], proba)

    def run():
        return fusion.refine_ref_view(*args, conf=0.5, rule=rule)
    for _ in range(3):
        run()
    ts = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        run()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(repeats):
            run()
        torch.cuda.synchronize()
    ks = [e.time_range.elapsed_us() / 1e3 for e in prof.events()
          if "geo_fuse_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
    if len(ks) != repeats:
        raise RuntimeError(f"profiler saw {len(ks)} fusion kernels, expected {repeats}")
    return statistics.median(ks), statistics.median(ts)


def surface_distance(p):
    """Distance of points (N,3) to the analytic scene: the sphere and the square of its plane."""
    p = p.double()
    d_sph = (p.norm(dim=1) - RADIUS).abs()
    qx = (p[:, 0].abs() - 3 * RADIUS).clamp(min=0)
    qy = (p[:, 1].abs() - 3 * RADIUS).clamp(min=0)
    d_pl = torch.sqrt(qx * qx + qy * qy + (p[:, 2] + RADIUS) ** 2)
    return torch.minimum(d_sph, d_pl)


def quality(views, label, taus, name, power, device):
    metas, depths, probas, images, proj = scan_inputs(views, 10, 7, device)
    surf = torch.cat([v["points"].to(device) for v in views])
    surf = surf[torch.randperm(len(surf), generator=torch.Generator().manual_seed(0))[:4_000_000].to(device)]
    lo = (surf.min(0).values - 10).double().cpu().numpy()
    hi = (surf.max(0).values + 10).double().cpu().numpy()
    for rule in fusion.RULES:
        xyz, _ = fusion.fuse_scan(metas, depths, probas, images, proj, conf=0.5, rule=rule)
        row = dict(bench="quality", scene=label, views=len(views), rule=rule, kept=len(xyz),
                   gpu=name, power_limit=power)
        err = surface_distance(xyz)
        for tau in taus:
            comp = dtu_eval.capped_nn(surf.float().contiguous(), xyz.contiguous(), lo, hi, cap=4 * tau,
                                      cell=2 * tau)
            row[f"accuracy_share_tau{tau:g}"] = round(float((err <= tau).double().mean()), 4)
            row[f"completeness_share_tau{tau:g}"] = round(float((comp <= tau).double().mean()), 4)
        print(json.dumps(row), flush=True)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--scan_views", type=int, default=150)
    ap.add_argument("--taus", nargs="+", type=float, default=[1.0, 2.0])
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_fusion.py needs a GPU")
    dev = "cuda:0"
    name, power = card()
    for W, H in ((1152, 864), (1920, 1056)):
        S = 10
        for rule in fusion.RULES:
            ms, call_ms = time_view(rule, W, H, S, a.repeats, dev)
            nbytes = bytes_per_pixel(S) * W * H
            print(json.dumps(dict(bench="view", rule=rule, wh=[W, H], S=S, kernel_ms=round(ms, 4),
                                  call_ms=round(call_ms, 4),
                                  counted_bytes=nbytes, counted_tbps=round(nbytes / ms / 1e9, 3),
                                  share_of_hbm=round(nbytes / (ms * 1e-3) / HBM_BPS, 3),
                                  repeats=a.repeats, gpu=name, power_limit=power)), flush=True)
        torch.cuda.empty_cache()

    views = synth_scenes.sphere_scene(a.scan_views, (1152, 864), seed=2, radius=RADIUS, device=dev)
    metas, depths, probas, images, proj = scan_inputs(views, 10, 3, dev)
    for v in views:
        del v["points"]
    for rule in fusion.RULES:
        fusion.fuse_scan(metas[:4], depths, probas, images, proj, conf=0.5, rule=rule)
        ts, n = [], 0
        for _ in range(3):
            torch.cuda.synchronize()
            a0, b0 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a0.record()
            xyz, _ = fusion.fuse_scan(metas, depths, probas, images, proj, conf=0.5, rule=rule)
            b0.record()
            torch.cuda.synchronize()
            ts.append(a0.elapsed_time(b0))
            n = len(xyz)
        print(json.dumps(dict(bench="fuse_scan", rule=rule, views=a.scan_views, wh=[1152, 864], S=10,
                              ms=round(statistics.median(ts), 2), kept=n, repeats=3, gpu=name,
                              power_limit=power)), flush=True)
    del views, metas, depths, probas, images, proj
    torch.cuda.empty_cache()

    quality(synth_scenes.sphere_scene(60, (1152, 864), seed=4, radius=RADIUS, device=dev),
            "sphere_60_views", a.taus, name, power, dev)
    quality(synth_scenes.sphere_scene(12, (1152, 864), seed=4, radius=RADIUS, device=dev),
            "sphere_12_views_thinned", a.taus, name, power, dev)


if __name__ == "__main__":
    main()
