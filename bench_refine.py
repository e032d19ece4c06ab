"""Time mesh refinement on the GPU (refine.py), and with --study measure what it does to a mesh's
error against a known surface.

Speed: bench_mesh.py's TSDF meshes of synth_scenes.sphere_scene at 49 and 150 views of 1152x864,
and the 49-view mesh decimated to 10 %, refined against those views (their float colours rounded
to uint8; each view's sources are the 10 views whose camera centres lie nearest, nearest first).
Each phase of each iteration (visibility, selection, sweep, smoothing) is timed with CUDA events;
one full untimed run per scene comes first (warm-up).  Peak device memory is torch's
max_memory_allocated over one refine_mesh call.

Study: synth_scenes.make_colmap(textured=True) renders views of its analytic height field
z = depth + 0.05 depth sin(3x / depth) cos(2y / depth).  Each view's sources are the other views
of the same camera (make_colmap draws the texture at each camera's own scale) in order of
decreasing angle between the cameras (the widest baselines first).  Meshes: the TSDF
mesh of the ground-truth depths times (1 + NOISE N(0, 1)) (seeded), that mesh decimated to 10 %,
the Poisson mesh at depth 8 of the noisy depths' points, and the TSDF mesh of the exact depths.
The error of a vertex is its first-order distance to the height field, |z - h(x, y)| /
sqrt(1 + |grad h|^2), in footprints (mesh.pixel_footprint of view 0's ground truth); RMS and p90
over the vertices before and after refinement.  Every line names the card and its power limit.

    python bench_refine.py [--views 49 150] [--wh 1152 864] [--repeats 3]
    python bench_refine.py --study [--study_views 12] [--study_wh 640 512]
"""
import argparse
import json
import subprocess

import numpy as np
import torch

from casmvsnet_pl_b200 import mesh, refine, simplify, synth_scenes

NOISE = 0.003
DEPTH = 3.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def timed(v, c, f, images, Ps, sources):
    """One refine_mesh call -> (per-iteration phase times in ms, stats, peak bytes)."""
    events = []

    def mark(phase):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        events.append((phase, e))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    mark("start")
    _, _, _, st = refine.refine_mesh(v, c, f, images, Ps, sources, log=lambda *a: None, mark=mark)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    phases = [dict() for _ in range(st["iterations"])]
    it = 0
    for (_, a), (name, b) in zip(events, events[1:]):
        phases[it][name] = a.elapsed_time(b)
        if name == "smoothing":
            it += 1
    return phases, st, peak


def nearest_sources(Ps, n=10):
    C = np.stack([refine.texture.eye_of(P) for P in Ps])
    d = np.linalg.norm(C[:, None] - C[None], axis=2)
    return [[int(j) for j in np.argsort(d[i], kind="stable") if j != i][:n] for i in range(len(Ps))]


def speed(a, name, power):
    for n in a.views:
        views = synth_scenes.sphere_scene(n, tuple(a.wh), seed=a.seed, device="cuda:0")
        Ps = [x["P"] for x in views]
        voxel = mesh.default_voxel_size([x["depth"] for x in views], Ps)
        v, c, f, _ = mesh.mesh_views([x["points"] for x in views], [x["depth"] for x in views],
                                     [x["image"] for x in views], Ps, voxel)
        images = [x["image"].round().clamp(0, 255).to(torch.uint8).contiguous() for x in views]
        del views
        sources = nearest_sources(Ps)
        scenes = [(f"tsdf_{n}", v, c, f)]
        if n == 49:
            dv, dc, df, _ = simplify.simplify_mesh(v, c, f, len(f) // 10, log=lambda *x: None)
            scenes.append((f"tsdf_{n}_decimated_10pct", dv, dc, df))
        for label, sv, sc, sf in scenes:
            timed(sv, sc, sf, images, Ps, sources)                      # warm-up
            runs = [timed(sv, sc, sf, images, Ps, sources) for _ in range(a.repeats)]
            per = {}
            for it in range(len(runs[0][0])):
                for ph in ("visibility", "selection", "sweep", "smoothing"):
                    per[f"it{it}_{ph}_ms"] = round(float(np.median([r[0][it][ph] for r in runs])), 3)
            total = float(np.median([sum(sum(p.values()) for p in r[0]) for r in runs]))
            st = runs[0][1]
            print(json.dumps(dict(scene=label, views=n, wh=a.wh, vertices=len(sv), faces=len(sf),
                                  **per, total_ms=round(total, 3), peak_bytes=int(runs[0][2]),
                                  seen=[s["seen"] for s in st["per_iteration"]],
                                  confident=[s["confident"] for s in st["per_iteration"]],
                                  repeats=a.repeats, gpu=name, power_limit=power)), flush=True)
        del images
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------- quality study
def surface_error(verts, rho):
    """First-order distance of each vertex to the height field, in footprints."""
    x = verts.double().cpu().numpy()
    a, b = 3.0 / DEPTH, 2.0 / DEPTH
    h = DEPTH + 0.05 * DEPTH * np.sin(a * x[:, 0]) * np.cos(b * x[:, 1])
    hx = 0.05 * DEPTH * a * np.cos(a * x[:, 0]) * np.cos(b * x[:, 1])
    hy = -0.05 * DEPTH * b * np.sin(a * x[:, 0]) * np.sin(b * x[:, 1])
    return np.abs(x[:, 2] - h) / np.sqrt(1 + hx * hx + hy * hy) / rho


def study_views(a, tmp):
    from PIL import Image

    from casmvsnet_pl_b200 import colmap
    model, depths = synth_scenes.make_colmap(tmp, n_views=a.study_views, image_wh=tuple(a.study_wh),
                                             depth=DEPTH, seed=a.seed, textured=True)
    rng = np.random.default_rng(a.seed)
    views = []
    for q, t, cid, nm in sorted(model.images.values(), key=lambda r: r[3]):
        cam, w, h, prm = model.cameras[cid]
        v = int(nm[len("view_"):-len(".png")])
        P = np.eye(4)
        P[:3, :3] = colmap.intrinsics(cam, prm)
        E = np.eye(4)
        E[:3, :3], E[:3, 3] = colmap.qvec_to_rotmat(q), t
        P = (P @ E).astype(np.float32)
        img = np.asarray(Image.open(f"{tmp}/images/{nm}").convert("RGB"))
        views.append(dict(v=v, P=P, image=img, depth=depths[v]))
    views.sort(key=lambda r: r["v"])
    for x in views:
        x["noisy"] = x["depth"] * (1 + NOISE * rng.standard_normal(x["depth"].shape))
    return views


def _points(depth, P):
    H, W = depth.shape
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    Pi = np.linalg.inv(P.astype(np.float64))
    q = np.stack([xs * depth, ys * depth, depth, np.ones_like(depth)], -1) @ Pi.T
    return q[..., :3] / q[..., 3:]


def tsdf(views, key, voxel):
    dev = "cuda:0"
    pts = [torch.from_numpy(_points(x[key], x["P"]).reshape(-1, 3)).float().to(dev) for x in views]
    vol = mesh.TSDFVolume(pts, voxel)
    for size in sorted({x[key].shape for x in views}):
        g = [x for x in views if x[key].shape == size]
        vol.integrate([torch.from_numpy(x[key]).float().to(dev) for x in g],
                      [torch.from_numpy(x["image"]).float().to(dev) for x in g], [x["P"] for x in g])
    return vol.extract()


def study(a, name, power):
    import tempfile

    from casmvsnet_pl_b200 import poisson
    with tempfile.TemporaryDirectory() as tmp:
        views = study_views(a, tmp)
    Ps = [x["P"] for x in views]
    rho = mesh.pixel_footprint(torch.from_numpy(views[0]["depth"]), Ps[0])
    C = np.stack([refine.texture.eye_of(P) for P in Ps])
    axis = (np.array([0.0, 0.0, DEPTH]) - C) / np.linalg.norm(np.array([0.0, 0.0, DEPTH]) - C, axis=1)[:, None]
    ang = np.arccos(np.clip(axis @ axis.T, -1, 1))
    # make_colmap renders its texture at a frequency set by each camera's focal length, so views of
    # the two cameras (even and odd views) show different textures: sources share the camera
    sources = [[int(j) for j in np.argsort(-ang[i], kind="stable") if j != i and (j - i) % 2 == 0]
               for i in range(len(Ps))]
    images = [torch.from_numpy(x["image"].copy()).cuda() for x in views]
    voxel = 2 * rho
    meshes = {}
    meshes["tsdf_noisy"] = tsdf(views, "noisy", voxel)
    v, c, f = meshes["tsdf_noisy"]
    meshes["tsdf_noisy_decimated_10pct"] = simplify.simplify_mesh(v, c, f, len(f) // 10,
                                                                  log=lambda *x: None)[:3]
    pts = torch.cat([torch.from_numpy(_points(x["noisy"], x["P"]).reshape(-1, 3)).float() for x in views]).cuda()
    cols = torch.cat([torch.from_numpy(x["image"].reshape(-1, 3)) for x in views]).cuda()
    meshes["poisson_noisy_depth8"] = poisson.poisson_mesh(pts, cols, cam_centres=C, depth=8,
                                                          log=lambda *x: None)[:3]
    meshes["tsdf_exact"] = tsdf(views, "depth", voxel)
    for label, (v, c, f) in meshes.items():
        e0 = surface_error(v, rho)
        rv, _, _, st = refine.refine_mesh(v, c, f, images, Ps, sources, log=lambda *x: None)
        e1 = surface_error(rv, rho)
        print(json.dumps(dict(study=label, views=len(views), wh=a.study_wh, vertices=len(v),
                              faces=len(f), footprint=rho, noise=NOISE,
                              rms_before=round(float(np.sqrt(np.mean(e0 ** 2))), 4),
                              rms_after=round(float(np.sqrt(np.mean(e1 ** 2))), 4),
                              p90_before=round(float(np.percentile(e0, 90)), 4),
                              p90_after=round(float(np.percentile(e1, 90)), 4),
                              seen=[s["seen"] for s in st["per_iteration"]],
                              confident=[s["confident"] for s in st["per_iteration"]],
                              mean_score=[round(s["mean_score"], 4) for s in st["per_iteration"]],
                              gpu=name, power_limit=power)), flush=True)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", nargs="+", type=int, default=[49, 150])
    ap.add_argument("--wh", nargs=2, type=int, default=[1152, 864])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--study", action="store_true", help="run the quality study instead")
    ap.add_argument("--study_views", type=int, default=12)
    ap.add_argument("--study_wh", nargs=2, type=int, default=[640, 512])
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_refine.py needs a GPU")
    name, power = card()
    (study if a.study else speed)(a, name, power)


if __name__ == "__main__":
    main()
