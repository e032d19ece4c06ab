"""The reference's eval.py end to end on the H100 engine (SURVEY.md 8 f-3 / f-4 callers):

    step 1 (eval.py:198-243)  depth + confidence for every reference view of a scan
    step 2 (eval.py:245-353)  geometric filter, refinement, fusion, PLY
    step 3 (optional)         DTU scores of the fused cloud (dtu_eval, evaluations/dtu/*.m),
                              straight from the device tensors when --dtu_gt is given

over the DTU *test* layout the reference reads (datasets/dtu.py:31-75,150-166, eval.py:76-98):

    <root>/Cameras/pair.txt, <root>/Cameras/{vid:08d}_cam.txt,
    <root>/Rectified/<scan>/rect_{vid+1:03d}_3_r5000.png

Everything between decoding the PNGs and writing the PLY stays on the GPU: images are uploaded as
bytes and normalised by casmvs_normalize_u8_fwd, depth maps never pass through PFM files unless
`depth_dir` is given (then the reference's depth_XXXX.pfm / proba_XXXX.pfm are written as well).

    python -m casmvsnet_pl_b200.eval_pipeline --root_dir DTU --scan scan1 --ckpt ckpt.ckpt [--dtu_gt GT]
"""
from __future__ import annotations

import argparse
import json
import os

import numpy as np
import torch

from . import fusion, io


def read_image_rgb_u8(path, img_wh):
    """cv2.imread + cv2.resize(INTER_LINEAR) + BGR->RGB (eval.py:76-79, 267-268) -> (H,W,3) uint8.
    (The reference's *network input* goes through PIL's BILINEAR resize, datasets/dtu.py:160-162;
    both decoders are host-side third-party code and are used as the reference uses them.)"""
    import cv2
    img = cv2.imread(path)
    if img is None:
        raise FileNotFoundError(path)
    return np.ascontiguousarray(cv2.resize(img, tuple(img_wh), interpolation=cv2.INTER_LINEAR)[:, :, ::-1])


def read_network_image_u8(path, img_wh):
    """PIL open + resize(BILINEAR) (datasets/dtu.py:159-162) -> (H,W,3) uint8 RGB."""
    from PIL import Image
    img = Image.open(path).convert("RGB")
    if img.size != tuple(img_wh):
        img = img.resize(tuple(img_wh), Image.BILINEAR)
    return np.ascontiguousarray(np.asarray(img, dtype=np.uint8))


class DTUTestScan:
    """Metas, per-view projection pyramids and image paths of one scan (datasets/dtu.py test mode)."""

    def __init__(self, root_dir, scan, img_wh=(1152, 864), n_views=5, levels=3, full_wh=(1600, 1200)):
        assert img_wh[0] % 32 == 0 and img_wh[1] % 32 == 0, "img_wh must both be multiples of 32!"
        self.root_dir, self.scan, self.img_wh, self.n_views = root_dir, scan, tuple(img_wh), n_views
        self.metas = io.read_pair_file(os.path.join(root_dir, "Cameras", "pair.txt"))
        self.proj_mats, self.depth_min = {}, {}
        vids = sorted({r for r, _ in self.metas} | {s for _, ss in self.metas for s in ss})
        for vid in vids:
            K, E, dmin = io.read_cam_file(os.path.join(root_dir, "Cameras", f"{vid:08d}_cam.txt"))
            self.proj_mats[vid] = io.pyramid_proj_mats(K, E, levels, self.img_wh, full_wh)
            self.depth_min[vid] = dmin

    def image_path(self, vid):
        return os.path.join(self.root_dir, "Rectified", self.scan, f"rect_{vid + 1:03d}_3_r5000.png")

    def views(self, device):
        """yields (ref_vid, imgs (V,3,H,W) float32 on `device`, proj_mats (V-1,levels,3,4) host)."""
        for ref, srcs in self.metas:
            ids = [ref] + srcs[: self.n_views - 1]
            u8 = np.stack([read_network_image_u8(self.image_path(v), self.img_wh) for v in ids])
            imgs = io.normalize_images(torch.from_numpy(u8).pin_memory(), device)
            yield ref, imgs, io.relative_proj_mats(self.proj_mats, ids)


@torch.no_grad()
def run_scan(model, scan: DTUTestScan, depth_interval=2.65, conf=0.999, min_geo_consistent=5,
             skip=1, max_ref_views=400, device="cuda:0", depth_dir=None, ply_path=None,
             dtu_gt=None, dtu_seed=0):
    """-> (xyz (N,3) float32, rgb (N,3) uint8) CUDA tensors; optional PFM / PLY outputs.
    With `dtu_gt` (a DTU ground-truth directory) the fused cloud is also scored by
    dtu_eval.evaluate_scan from the device tensors, the scores are written next to the PLY as
    <ply>_scores.json when ply_path is given, and (xyz, rgb, scores) is returned."""
    depths, probas = {}, {}
    writer = io.DepthWriter(depth_dir) if depth_dir else None
    for ref, imgs, pm in scan.views(device):
        res = model(imgs.unsqueeze(0), pm.unsqueeze(0).to(device), scan.depth_min[ref], depth_interval)
        depths[ref] = torch.nan_to_num(res["depth_0"][0]).clone()            # eval.py:224-227
        probas[ref] = torch.nan_to_num(res["confidence_2"][0]).clone()
        if writer:
            writer(scan.scan, ref, depths[ref].cpu().numpy(), probas[ref].cpu().numpy())
    images = {v: torch.from_numpy(read_image_rgb_u8(scan.image_path(v), scan.img_wh)).to(device).float()
              for v in depths}
    proj0 = {v: scan.proj_mats[v][0].numpy() for v in scan.proj_mats}     # finest level (eval.py:108)
    xyz, rgb = fusion.fuse_scan(scan.metas, depths, probas, images, proj0, conf, min_geo_consistent,
                                skip, max_ref_views)
    if ply_path:
        fusion.write_ply(ply_path, xyz, rgb)
    if dtu_gt is None:
        return xyz, rgb
    from . import dtu_eval
    scores = dtu_eval.evaluate_scan(xyz, dtu_eval.scan_number(scan.scan), dtu_gt, seed=dtu_seed)
    if ply_path:
        with open(os.path.splitext(ply_path)[0] + "_scores.json", "w") as f:
            json.dump(scores, f, indent=1)
    return xyz, rgb, scores


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root_dir", required=True)
    ap.add_argument("--scan", required=True)
    ap.add_argument("--ckpt", default="")
    ap.add_argument("--img_wh", nargs=2, type=int, default=[1152, 864])
    ap.add_argument("--n_views", type=int, default=5)
    ap.add_argument("--n_depths", nargs="+", type=int, default=[8, 32, 48])
    ap.add_argument("--interval_ratios", nargs="+", type=float, default=[1.0, 2.0, 4.0])
    ap.add_argument("--num_groups", type=int, default=1)
    ap.add_argument("--depth_interval", type=float, default=2.65)
    ap.add_argument("--conf", type=float, default=0.999)
    ap.add_argument("--min_geo_consistent", type=int, default=5)
    ap.add_argument("--skip", type=int, default=1)
    ap.add_argument("--precision", default="tf32", choices=["fp32", "tf32"])
    ap.add_argument("--out", default="results/dtu")
    ap.add_argument("--dtu_gt", default=None, help="DTU ground-truth directory: score the fused cloud")
    ap.add_argument("--dtu_seed", type=int, default=0)
    a = ap.parse_args()
    from . import ABN
    from .models.mvsnet import CascadeMVSNet
    model = CascadeMVSNet(n_depths=a.n_depths, interval_ratios=a.interval_ratios,
                          num_groups=a.num_groups, norm_act=ABN, precision=a.precision)
    if a.ckpt:
        sd = torch.load(a.ckpt, map_location="cpu")
        sd = sd.get("state_dict", sd)
        sd = {k[len("model."):] if k.startswith("model.") else k: v for k, v in sd.items()}   # utils:57-59
        model.load_state_dict(sd)
    model = model.eval().cuda()
    scan = DTUTestScan(a.root_dir, a.scan, tuple(a.img_wh), a.n_views)
    os.makedirs(os.path.join(a.out, "points"), exist_ok=True)
    out = run_scan(model, scan, a.depth_interval, a.conf, a.min_geo_consistent, a.skip,
                   depth_dir=os.path.join(a.out, "depth"),
                   ply_path=os.path.join(a.out, "points", f"{a.scan}.ply"), dtu_gt=a.dtu_gt,
                   dtu_seed=a.dtu_seed)
    print(f"{a.scan} contains {len(out[0]) / 1e6:.2f} M points")
    if a.dtu_gt is not None:
        from .dtu_eval import _fmt
        print(_fmt(out[2]))


if __name__ == "__main__":
    main()
