"""Photometric loss (csrc/photo_loss.cu) timings: forward + backward at 640x512 (V = 3, K = 1)
and 1152x864 (V = 5, K = 2) for B = 1 and 2, its counted bytes over kernel time against the
H100 SXM's 3.35 TB/s, the same loss as a float32 torch autograd restatement (grid_sample,
pooling, topk) for comparison, and one 640x512 training step with sl1 and with photo.

    python bench_photo_loss.py [--iters 50]
    python bench_photo_loss.py --study      # fine-tuning study on a textured synthetic capture

Counted bytes per level (the least traffic the rule needs): forward reads the reference and S
source images (3 floats per pixel each, at the level's pixels) and the depth, and writes the
selection (2 bytes); backward reads the same plus the selection and writes the gradient.  The
strided level subsample and the bilinear taps touch more sectors than that, so the ratio is a
lower bound on the achieved bandwidth."""
import argparse
import json
import subprocess

import torch
import torch.nn.functional as F

from casmvsnet_pl_b200 import io, losses, synth, train

RATIOS = [1.0, 2.0, 4.0]
HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def make(B, V, W, H, seed=0):
    g = torch.Generator().manual_seed(seed)
    u8 = torch.randint(0, 256, (B * V, H, W, 3), generator=g, dtype=torch.uint8)
    imgs = io.normalize_images(u8.cuda()).view(B, V, 3, H, W)
    pm = synth.projection_matrices(V, W, H, 3).unsqueeze(0).expand(B, -1, -1, -1, -1).contiguous().cuda()
    ds = [(synth.CONVERGE_MM + 20 * torch.rand(B, H >> l, W >> l, generator=g)).cuda() for l in range(3)]
    return imgs, pm, ds, torch.full((B, 1), 2.65, device="cuda")


def counted_bytes(B, V, W, H):
    fwd = bwd = 0
    for l in range(3):
        n = B * (H >> l) * (W >> l)
        fwd += n * (V * 3 * 4 + 4 + 2)
        bwd += n * (V * 3 * 4 + 4 + 2 + 4)
    return fwd, bwd


def torch_photo(ds, imgs, pm, dint, K, lam):
    """The rule in float32 torch autograd: grid_sample warps, 3x3 avg_pool SSIM, topk."""
    B, V, _, H, W = imgs.shape
    mean = torch.tensor(io.IMAGENET_MEAN, device=imgs.device).view(1, 1, 3, 1, 1)
    std = torch.tensor(io.IMAGENET_STD, device=imgs.device).view(1, 1, 3, 1, 1)
    total = 0.0
    for l, d in enumerate(ds):
        I = (imgs * std + mean)[..., :: 1 << l, :: 1 << l]
        h, w = I.shape[-2:]
        ref, src = I[:, 0], I[:, 1:]
        ys, xs = torch.meshgrid(torch.arange(h, device=d.device, dtype=torch.float32),
                                torch.arange(w, device=d.device, dtype=torch.float32), indexing="ij")
        P = pm[:, :, l]
        pix = torch.stack([xs, ys, torch.ones_like(xs)], 0).view(1, 1, 3, -1)
        p = P[..., :3] @ pix + P[..., 3:] / d.view(B, 1, 1, -1)
        z = p[:, :, 2]
        u, v = p[:, :, 0] / z, p[:, :, 1] / z
        ok = (z > 1e-7) & (u >= 0) & (u <= w - 1) & (v >= 0) & (v <= h - 1)
        grid = torch.stack([u / (w - 1) * 2 - 1, v / (h - 1) * 2 - 1], -1).view(B * (V - 1), h, w, 2)
        y = F.grid_sample(src.reshape(B * (V - 1), 3, h, w), grid, align_corners=True).view(B, V - 1, 3, h, w)
        x = ref[:, None].expand_as(y).reshape(-1, 3, h, w)
        yy = y.reshape(-1, 3, h, w)
        pool = lambda t: F.avg_pool2d(t, 3, 1)                       # noqa: E731
        mx, my = pool(x), pool(yy)
        sxx, syy, sxy = pool(x * x) - mx * mx, pool(yy * yy) - my * my, pool(x * yy) - mx * my
        ssim = (2 * mx * my + 1e-4) * (2 * sxy + 9e-4) / ((mx * mx + my * my + 1e-4) * (sxx + syy + 9e-4))
        l1 = (x - yy).abs()[..., 1:-1, 1:-1]
        e = (0.85 * (1 - ssim) / 2 + 0.15 * l1).mean(1).view(B, V - 1, h - 2, w - 2)
        okw = -F.max_pool2d(-ok.view(B * (V - 1), 1, h, w).float(), 3, 1).view(B, V - 1, h - 2, w - 2) > 0
        e = torch.where(okw, e, torch.full_like(e, 1e4))
        best = torch.topk(e, K, dim=1, largest=False).values
        valid = best < 1e4
        loss_q = torch.where(valid, best, torch.zeros_like(best)).sum(1) / valid.sum(1).clamp(min=1)
        has = valid[:, 0]
        P_l = loss_q[has].sum() / has.sum().clamp(min=1)
        dh = d / (dint.view(B, 1, 1) * RATIOS[l])
        gx = (ref[..., 1:] - ref[..., :-1]).abs().mean(1)
        gy = (ref[..., 1:, :] - ref[..., :-1, :]).abs().mean(1)
        S_l = ((dh[..., 1:] - dh[..., :-1]).abs() * torch.exp(-gx)).mean() + \
            ((dh[..., 1:, :] - dh[..., :-1, :]).abs() * torch.exp(-gy)).mean()
        total = total + 2.0 ** (1 - l) * (P_l + lam * S_l)
    return total


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench_loss(B, V, W, H, K, iters):
    imgs, pm, ds, dint = make(B, V, W, H)
    params = [d.clone().requires_grad_(True) for d in ds]
    res = {f"depth_{l}": p for l, p in enumerate(params)}

    def ours():
        loss, _ = losses.photo_loss(res, imgs, pm, dint, RATIOS, 3, K)
        loss.backward()

    def fwd_only():
        with torch.no_grad():
            losses.photo_loss(res, imgs, pm, dint, RATIOS, 3, K)

    def ref():
        torch_photo(params, imgs, pm, dint, K, 0.01).backward()
    t_fb = timed(ours, iters)
    t_f = timed(fwd_only, iters)
    fb, bb = counted_bytes(B, V, W, H)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ours()
    torch.cuda.synchronize()
    peak_ours = torch.cuda.max_memory_allocated() - base
    t_ref = timed(ref, max(5, iters // 5))
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ref()
    torch.cuda.synchronize()
    peak_ref = torch.cuda.max_memory_allocated() - base
    return {"shape": f"{W}x{H}", "B": B, "V": V, "K": K, "fwd_ms": t_f, "fwd_bwd_ms": t_fb,
            "bwd_ms": t_fb - t_f, "fwd_counted_TBps": fb / (t_f * 1e-3) / 1e12,
            "fwd_share_of_hbm": fb / (t_f * 1e-3) / HBM,
            "bwd_share_of_hbm": bb / ((t_fb - t_f) * 1e-3) / HBM,
            "torch_fp32_fwd_bwd_ms": t_ref, "peak_MiB": peak_ours / 2 ** 20,
            "torch_fp32_peak_MiB": peak_ref / 2 ** 20}


def bench_step(loss_type, iters):
    from casmvsnet_pl_b200 import InPlaceABN
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    argv = ["--loss_type", loss_type, "--optimizer", "adam", "--train_list", "x", "--val_list", "y"]
    a = train.parse_args(argv)
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=InPlaceABN).cuda().train()
    imgs, pm, dmin, dint = synth.make_inputs(B=1, V=3, W=640, H=512, seed=0)
    s = {"imgs": imgs.cuda(), "proj_mats": pm.cuda(), "init_depth_min": torch.full((1, 1), dmin, device="cuda"),
         "depth_interval": torch.full((1, 1), dint, device="cuda"),
         "depths": {f"level_{l}": torch.full((1, 512 >> l, 640 >> l), 700.0, device="cuda") for l in range(3)},
         "masks": {f"level_{l}": torch.ones(1, 512 >> l, 640 >> l, dtype=torch.bool, device="cuda")
                   for l in range(3)}}
    tr = train.Trainer(a, model, "cuda")
    return {"step": loss_type, "ms": timed(lambda: tr.train_step(s), iters)}


def study(epochs=16, lams=(0.0, 0.01, 0.1)):
    """The network fine-tuned by train.py on one textured synthetic capture
    (synth_scenes.make_colmap textured=True, 8 views, 640x512, V = 5, K = 1, adam, lr 1e-3,
    --seed 0, so every run starts from the same initialisation), once per smoothness weight.
    Before and after: the level-0 depth of every reference view in eval mode against the
    float64 ground truth (synth_scenes.height_field_depth at the network size), as the mean
    |depth - gt| in depth intervals and the share of pixels within 4 intervals."""
    import os
    import tempfile

    from casmvsnet_pl_b200 import synth_scenes, train_data
    out = []
    with tempfile.TemporaryDirectory() as root:
        cap = os.path.join(root, "capture")
        synth_scenes.make_colmap(cap, n_views=8, image_wh=(640, 512), n_points=3000, seed=5, textured=True)
        ts = train_data.ColmapTrainSet(cap, n_views=5, img_wh=(640, 512), device="cuda", log=lambda m: None)
        sc = ts.scan.scene
        gts = []
        for ids in ts.ids:
            v = ids[0]
            K = sc.K[v].copy()
            K[0] *= 640 / sc.wh[v, 0]
            K[1] *= 512 / sc.wh[v, 1]
            gts.append(torch.from_numpy(synth_scenes.height_field_depth(K, sc.E[v], (640, 512))[0]).cuda())

        @torch.no_grad()
        def error(model):
            model.eval()
            err = within = 0.0
            for i, gt in enumerate(gts):
                s = ts.batch([i])
                d = model(s["imgs"], s["proj_mats"], s["init_depth_min"], s["depth_interval"])["depth_0"][0]
                e = (d.double() - gt).abs() / s["depth_interval"].item()
                err += e.mean().item() / len(gts)
                within += (e <= 4).double().mean().item() / len(gts)
            return {"mean_intervals": err, "within_4": within}

        argv = ["--dataset_name", "colmap", "--loss_type", "photo", "--root_dir", cap, "--img_wh", "640",
                "512", "--n_views", "5", "--num_epochs", str(epochs), "--optimizer", "adam", "--lr", "1e-3",
                "--seed", "0", "--log_every", "1000", "--num_workers", "0"]
        a = train.parse_args(argv)
        torch.manual_seed(0)
        before = error(train.build_model(a, "cuda"))
        here = os.getcwd()
        for lam in lams:
            os.chdir(root)
            try:
                trainer = train.main(argv + ["--smooth_weight", str(lam), "--exp_name", f"lam{lam}"])
            finally:
                os.chdir(here)
            out.append({"lambda": lam, "epochs": epochs, "steps": trainer.global_step, "before": before,
                        "after": error(trainer.model)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--study", action="store_true",
                    help="run the synthetic fine-tuning study only (train.py, three smoothness weights)")
    a = ap.parse_args()
    gpu = card()
    if a.study:
        for rec in study():
            print(json.dumps({"card": gpu, "study": rec}))
        return
    for B in (1, 2):
        for (W, H, V, K) in ((640, 512, 3, 1), (1152, 864, 5, 2)):
            print(json.dumps({"card": gpu, **bench_loss(B, V, W, H, K, a.iters)}))
    for lt in ("sl1", "photo"):
        print(json.dumps({"card": gpu, **bench_step(lt, max(5, a.iters // 5))}))


if __name__ == "__main__":
    main()
