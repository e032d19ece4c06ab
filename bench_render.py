"""Time headless rendering on the GPU at the sizes a user renders: the fused-cloud stand-in of an
analytic scene (a sphere on a plane, synth_scenes.sphere_scene: every surface pixel of 49 and 150
views of 1152x864) and its TSDF mesh (mesh.mesh_views at the default voxel), drawn at 1920x1080.

Cases per scene size: the cloud from the default view and from one scene camera (view 0, its
focal length scaled to the wider image), the mesh from the default view, and the mesh from a
close-up camera 1.5 radii from the sphere's centre, where triangles span many pixels.  Each
render call is timed with CUDA events, median of --repeats after one warm-up call.  The host side
of a command-line run (PLY read, upload, PNG encode) is timed with a host clock around work
that ends in a synchronise.  Prints one JSON line per case with the card name and power limit
read in the same run.

    python bench_render.py [--views 49 150] [--wh 1920 1080] [--repeats 5]
"""
import argparse
import io
import json
import os
import subprocess
import tempfile
import time

import numpy as np
import torch

from casmvsnet_pl_b200 import fusion, mesh, render, synth_scenes

SCENE_WH = (1152, 864)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def timed(fn, repeats):
    fn()                                                          # warm-up
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), out


def scene_camera(P, wh):
    """View P of the scene (f = 0.9 W, centred principal point at SCENE_WH) re-aimed at an image
    of size wh with the same f / W."""
    W0, H0 = SCENE_WH
    W, H = wh
    K0 = np.array([[0.9 * W0, 0, W0 / 2], [0, 0.9 * W0, H0 / 2], [0, 0, 1]])
    K1 = np.array([[0.9 * W, 0, W / 2 - 0.5], [0, 0.9 * W, H / 2 - 0.5], [0, 0, 1]])
    A = np.eye(4)
    A[:3, :3] = K1 @ np.linalg.inv(K0)
    return (A @ np.asarray(P, np.float64)).astype(np.float32)


def close_up(wh, dist=1.5):
    C = dist * np.array([np.cos(np.radians(35)) * np.cos(0.4), np.cos(np.radians(35)) * np.sin(0.4),
                         np.sin(np.radians(35))])
    R = synth_scenes._look_at(C, np.zeros(3))
    W, H = wh
    K = np.array([[0.9 * W, 0, W / 2 - 0.5], [0, 0.9 * W, H / 2 - 0.5], [0, 0, 1]])
    E = np.eye(4)
    E[:3, :3], E[:3, 3] = R, -R @ C
    return render.projection(K, E).astype(np.float32)


def host_side(xyz, rgb, image):
    """Seconds for the command line's host work on this cloud: PLY read, upload, PNG encode."""
    from PIL import Image
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "scan.ply")
        fusion.write_ply(path, xyz, rgb)
        t0 = time.perf_counter()
        x, c, _ = render.load_scan(path, False)
        t1 = time.perf_counter()
        xd, cd = torch.from_numpy(x).cuda(), torch.from_numpy(c).cuda()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        Image.fromarray(image).save(io.BytesIO(), format="png")
        t3 = time.perf_counter()
        mb = os.path.getsize(path) / 2 ** 20
        del xd, cd
    return dict(ply_mb=round(mb, 1), ply_read_s=round(t1 - t0, 3), upload_s=round(t2 - t1, 3),
                png_encode_s=round(t3 - t2, 3))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", nargs="+", type=int, default=[49, 150])
    ap.add_argument("--wh", nargs=2, type=int, default=[1920, 1080])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_render.py needs a GPU")
    name, power = card()
    wh = tuple(a.wh)
    for n in a.views:
        views = synth_scenes.sphere_scene(n, SCENE_WH, seed=a.seed, device="cuda:0")
        xyz = torch.cat([v["points"] for v in views])
        rgb = torch.cat([v["image"][v["depth"] > 0] for v in views]).round().to(torch.uint8)
        verts, cols, faces, st = mesh.mesh_views([v["points"] for v in views],
                                                 [v["depth"] for v in views],
                                                 [v["image"] for v in views], [v["P"] for v in views])
        P0 = views[0]["P"]
        for v in views:
            del v["depth"], v["image"], v["points"]
        torch.cuda.empty_cache()
        P_cloud = render.projection(*render.default_view(xyz, wh))
        P_mesh = render.projection(*render.default_view(verts, wh))
        P_scene, P_close = scene_camera(P0, wh), close_up(wh)
        cases = [
            ("cloud_default", lambda: render.render_points(xyz, rgb, P_cloud, wh)),
            ("cloud_scene_camera", lambda: render.render_points(xyz, rgb, P_scene, wh)),
            ("mesh_default", lambda: render.render_mesh(verts, cols, faces, P_mesh, wh)),
            ("mesh_close_up", lambda: render.render_mesh(verts, cols, faces, P_close, wh)),
        ]
        common = dict(views=n, points=len(xyz), triangles=len(faces), voxel=round(st["voxel"], 6),
                      wh=list(wh), repeats=a.repeats, gpu=name, power_limit=power)
        image = None
        for case, fn in cases:
            ms, (img, depth) = timed(fn, a.repeats)
            if case == "cloud_default":
                image = img.cpu().numpy()
            print(json.dumps(dict(case=case, ms=round(ms, 3), drawn=int((depth > 0).sum()), **common)),
                  flush=True)
        host = host_side(xyz.cpu().numpy(), rgb.cpu().numpy(), image)
        print(json.dumps(dict(case="cli_host_side", **host, **common)), flush=True)
        del views, xyz, rgb, verts, cols, faces
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
