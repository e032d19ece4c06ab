"""Time the seam levelling of mesh texturing on the GPU (texture.py, level=True) on
bench_texture.py's scene: a sphere on a plane seen by 49 views of 1152x864
(synth_scenes.sphere_scene), its full TSDF mesh and that mesh decimated to 10 % and 1 %.  The photos
are the scene's images rounded to uint8 once, then given seeded per-view, per-channel gains in
[0.75, 1.25] and biases in [-15, 15], so that the seams have steps to level.  Each phase is timed
with CUDA events in a run that follows one untimed warm-up run of the same mesh: seams (unknowns,
seam records, samples and pair colours), assembly (the CSR and right-hand side), solve (CG, with
its iterations) and apply (owners and the apply pass).  Prints one JSON line per mesh with the
texturing time without levelling, the peak allocation above what the mesh and photos hold, the
seam RMS before and after, the apply pass's bytes per second against 3.35 TB/s (the bytes the
owner and apply passes must move, counted below), and the card name and power limit read in the
same run.

    python bench_texture_level.py [--views 49] [--wh 1152 864] [--ratios 1 0.1 0.01]
"""
import argparse
import json

import numpy as np
import torch

from bench_mesh import card
from casmvsnet_pl_b200 import mesh, simplify, synth_scenes, texture

PHASES = ("seams", "assembly", "solve", "apply")
HBM_BYTES_PER_S = 3.35e12


def gained(photos, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for p in photos:
        gain = (0.75 + 0.5 * torch.rand(3, generator=g, dtype=torch.float64)).to(p.device)
        bias = (-15 + 30 * torch.rand(3, generator=g, dtype=torch.float64)).to(p.device)
        out.append((p.double() * gain + bias).round().clamp(0, 255).to(torch.uint8))
    return out


def apply_bytes(st):
    """The owner keys, 8 bytes per atlas texel: written once when they are cleared, read by the
    apply pass and by the count of adjusted texels; and 3 bytes read and 3 written per owned
    texel.  The owner pass's scattered atomics are not counted."""
    texels = st["pages"] * st["page_side"] ** 2
    return 8 * texels * 2 + 8 * texels + 6 * st["level"]["texels_adjusted"]


def run_once(v, c, f, photos, Ps):
    evs = []

    def mark(phase):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        evs.append((phase, e))

    torch.cuda.synchronize()
    uv, page, atlas, st = texture.texture_mesh(v, c, f, photos, Ps, mark=mark, level=True)
    torch.cuda.synchronize()
    ms = dict.fromkeys(PHASES, 0.0)
    fill = [e for p, e in evs if p == "fill"][-1]
    prev = fill
    for phase, e in evs:
        if phase in PHASES:
            ms[phase] += prev.elapsed_time(e)
            prev = e
    return ms, st


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--wh", nargs=2, type=int, default=[1152, 864])
    ap.add_argument("--ratios", nargs="+", type=float, default=[1.0, 0.1, 0.01])
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_texture_level.py needs a GPU")
    name, power = card()
    views = synth_scenes.sphere_scene(a.views, tuple(a.wh), seed=a.seed, device="cuda:0")
    voxel = mesh.default_voxel_size([x["depth"] for x in views], [x["P"] for x in views])
    v0, c0, f0, _ = mesh.mesh_views([x["points"] for x in views], [x["depth"] for x in views],
                                    [x["image"] for x in views], [x["P"] for x in views], voxel)
    photos = gained([x["image"].round().clamp(0, 255).to(torch.uint8) for x in views], a.seed + 1)
    Ps = [x["P"] for x in views]
    del views
    torch.cuda.empty_cache()
    for r in a.ratios:
        if r < 1:
            v, c, f, _ = simplify.simplify_mesh(v0, c0, f0, max(1, round(r * len(f0))))
        else:
            v, c, f = v0, c0, f0
        run_once(v, c, f, photos, Ps)                                     # warm-up
        torch.cuda.synchronize()
        s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s0.record()
        texture.texture_mesh(v, c, f, photos, Ps)
        s1.record()
        torch.cuda.synchronize()
        plain_ms = s0.elapsed_time(s1)
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        ms, st = run_once(v, c, f, photos, Ps)
        peak = torch.cuda.max_memory_allocated() - base
        lv = st["level"]
        nbytes = apply_bytes(st)
        print(json.dumps(dict(views=len(Ps), wh=a.wh, ratio=r, faces=len(f),
                              **{f"{k}_ms": round(val, 3) for k, val in ms.items()},
                              level_ms=round(sum(ms.values()), 3),
                              texture_without_level_ms=round(plain_ms, 3),
                              cg_iterations=lv["cg_iterations"], converged=lv["converged"],
                              cg_ratios=[float(f"{x:.3g}") for x in lv["cg_ratios"]],
                              unknowns=lv["unknowns"], seam_pairs=lv["seam_pairs"],
                              smoothing_edges=lv["smoothing_edges"], nnz=lv["nnz"],
                              texels_adjusted=lv["texels_adjusted"], pages=st["pages"],
                              page_side=st["page_side"],
                              seam_rms_before=round(lv["seam_rms_before"], 3),
                              seam_rms_after=round(lv["seam_rms_after"], 3),
                              peak_alloc_mib=round(peak / 2**20, 1),
                              apply_bytes=nbytes,
                              apply_tb_per_s=round(nbytes / (ms["apply"] * 1e-3) / 1e12, 3),
                              apply_share_of_hbm=round(nbytes / (ms["apply"] * 1e-3) / HBM_BYTES_PER_S, 3),
                              gpu=name, power_limit=power)), flush=True)
        del v, c, f
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
