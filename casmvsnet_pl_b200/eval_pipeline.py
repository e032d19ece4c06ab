"""The reference's eval.py end to end on the H100 engine (SURVEY.md 8 f-3 / f-4 callers):

    step 1 (eval.py:198-243)  depth + confidence for every reference view of a scan
    step 2 (eval.py:245-353)  geometric filter, refinement, fusion, PLY
    step 3 (optional)         DTU scores of the fused cloud (dtu_eval, evaluations/dtu/*.m),
                              straight from the device tensors when --dtu_gt is given

over the three test layouts eval.py reads (--dataset_name):

    dtu         DTUTestScan         datasets/dtu.py:31-75,150-166, eval.py:76-98
                <root>/Cameras/pair.txt, <root>/Cameras/{vid:08d}_cam.txt,
                <root>/Rectified/<scan>/rect_{vid+1:03d}_3_r5000.png
    tanks       TanksTestScan       datasets/tanks.py; <root>/<split>/<scan>/{pair.txt, cams, images}
    blendedmvs  BlendedMVSTestScan  datasets/blendedmvs.py; <root>/<scan>/{cams, blended_images,
                                    rendered_depth_maps}, scan lists in <root>/..

Everything between decoding the images and writing the PLY stays on the GPU.  DTU images are
decoded and resized on the host per use, as the reference does, uploaded as bytes and normalised
by casmvs_normalize_u8_fwd.  Tanks and BlendedMVS scans decode each view once into SceneImages,
which resizes on the device with kernels byte-identical to Pillow and cv2.  Depth maps never pass
through PFM files unless `depth_dir` is given (then the reference's depth_XXXX.pfm /
proba_XXXX.pfm are written as well).

    python -m casmvsnet_pl_b200.eval_pipeline --root_dir DTU --scan scan1 --ckpt ckpt.ckpt [--dtu_gt GT]
    python -m casmvsnet_pl_b200.eval_pipeline --dataset_name tanks --split intermediate --root_dir TNT
    python -m casmvsnet_pl_b200.eval_pipeline --dataset_name blendedmvs --split val \
        --root_dir BlendedMVS/dataset_low_res --img_wh 768 576
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

    def depth_range(self, ref, depth_interval):
        """(init_depth_min, depth_interval) of reference view `ref` (eval.py:188-190, 214-222)."""
        return self.depth_min[ref], depth_interval

    def fusion_images(self, vids, device):
        return {v: torch.from_numpy(read_image_rgb_u8(self.image_path(v), self.img_wh)).to(device).float()
                for v in vids}


def _decode_pil_cv2(path):
    """One view file decoded by both libraries the reference uses on it: PIL (network input,
    RGB) and cv2 (fusion colours, BGR turned RGB)."""
    import cv2
    from PIL import Image
    with Image.open(path) as im:
        pil = np.array(im.convert("RGB"), dtype=np.uint8)
    bgr = cv2.imread(path)
    if bgr is None:
        raise FileNotFoundError(path)
    return pil, np.ascontiguousarray(bgr[:, :, ::-1])


class SceneImages:
    """Every view image of a scan decoded once and kept, resized, in device memory:
    `net` (n,h,w,3) uint8 = PIL decode + Image.resize(img_wh, BILINEAR) (the network input) and
    `fus` (n,h,w,3) uint8 RGB = cv2.imread + cv2.resize(INTER_LINEAR) (the fusion colours).
    Decoding runs in a small host thread pool while the device resizes the views already
    uploaded (io.resize_u8_pil / io.resize_u8_linear, byte-identical to Pillow / cv2).  A view
    is decoded once instead of once per reference view it takes part in, plus once for fusion."""

    def __init__(self, paths, img_wh, device, workers=4):
        from concurrent.futures import ThreadPoolExecutor
        self.index = {v: i for i, v in enumerate(paths)}
        w, h = img_wh
        n = len(self.index)
        self.net = torch.empty(n, h, w, 3, dtype=torch.uint8, device=device)
        self.fus = torch.empty(n, h, w, 3, dtype=torch.uint8, device=device)
        with ThreadPoolExecutor(max(1, workers)) as ex:
            for i, (pil, bgr) in enumerate(ex.map(_decode_pil_cv2, paths.values())):
                io.resize_u8_pil(torch.from_numpy(pil).pin_memory().to(device, non_blocking=True)[None],
                                 img_wh, out=self.net[i:i + 1])
                io.resize_u8_linear(torch.from_numpy(bgr).pin_memory().to(device, non_blocking=True)[None],
                                    img_wh, out=self.fus[i:i + 1])

    def network(self, ids):
        """(V,3,h,w) float32: ToTensor + Normalize of views `ids`, gathered from the cache."""
        idx = torch.tensor([self.index[v] for v in ids], device=self.net.device)
        return io.normalize_images(self.net.index_select(0, idx))

    def fusion(self, vid):
        return self.fus[self.index[vid]].float()


class _CachedScan:
    """Shared part of the Tanks and BlendedMVS readers: per-view images come from SceneImages,
    built on the first views() call.  host_images=True instead decodes and resizes every image
    on the host each time it is used, as the reference does (its PIL / cv2 route, kept as the
    reference the device route is tested and timed against)."""
    host_images = False
    _images = None

    def _image_cache(self, device):
        if self._images is None:
            self._images = SceneImages({v: self.image_path(v) for v in self.proj_mats}, self.img_wh,
                                       device)
        return self._images

    def views(self, device):
        """yields (ref_vid, imgs (V,3,H,W) float32 on `device`, proj_mats (V-1,levels,3,4) host)."""
        cache = None if self.host_images else self._image_cache(device)
        for ref, srcs in self.metas:
            ids = [ref] + srcs[: self.n_views - 1]
            if cache is None:
                u8 = np.stack([read_network_image_u8(self.image_path(v), self.img_wh) for v in ids])
                imgs = io.normalize_images(torch.from_numpy(u8).pin_memory(), device)
            else:
                imgs = cache.network(ids)
            yield ref, imgs, io.relative_proj_mats(self.proj_mats, ids)

    def fusion_images(self, vids, device):
        if self.host_images:
            return DTUTestScan.fusion_images(self, vids, device)
        cache = self._image_cache(device)
        return {v: cache.fusion(v) for v in vids}


def _read_proj_mats(cam_path, vids, img_wh, full_wh, levels, scale=None):
    """build_proj_mats of datasets/tanks.py:76-99 / blendedmvs.py:58-104 -> (proj_mats, depth_min)
    per view.  `scale` (BlendedMVS): None, or a one-element list holding the scan's depth scale
    factor (100 / depth_min of the first cam read, set here when empty), applied to depth_min and
    to the extrinsic translation (blendedmvs.py:98-103)."""
    proj, dmin = {}, {}
    for vid in vids:
        K, E, d = io.read_cam_file(cam_path(vid))
        if scale is not None:
            if not scale:
                scale.append(100 / d)
            d *= scale[0]
            E[:3, 3] *= scale[0]
        proj[vid] = io.pyramid_proj_mats(K, E, levels, img_wh, full_wh)
        dmin[vid] = d
    return proj, dmin


class TanksTestScan(_CachedScan):
    """One Tanks and Temples scan in the layout datasets/tanks.py reads (test mode):

        <root>/<split>/<scan>/pair.txt, cams/{vid:08d}_cam.txt, images/{vid:08d}.jpg

    Intrinsics are scaled by img_wh / native size / 4 with the scan's native image size
    (tanks.py:34-58, 86-87); depth_min comes from each view's cam file and the depth interval from
    the reference's hand-tuned per-scan table (tanks.py:42-64), so run_scan's depth_interval has
    no effect, as in the reference.  Every view of pair.txt is a reference view."""
    SCANS = {
        "intermediate": {"Family": ((1920, 1080), 2.5e-3), "Francis": ((1920, 1080), 1e-2),
                         "Horse": ((1920, 1080), 1.5e-3), "Lighthouse": ((2048, 1080), 1.5e-2),
                         "M60": ((2048, 1080), 5e-3), "Panther": ((2048, 1080), 5e-3),
                         "Playground": ((1920, 1080), 7e-3), "Train": ((1920, 1080), 5e-3)},
        "advanced": {"Auditorium": ((1920, 1080), 3e-2), "Ballroom": ((1920, 1080), 2e-2),
                     "Courtroom": ((1920, 1080), 2e-2), "Museum": ((1920, 1080), 2e-2),
                     "Palace": ((1920, 1080), 1e-2), "Temple": ((1920, 1080), 1e-2)},
    }

    def __init__(self, root_dir, split, scan, img_wh=(1152, 864), n_views=5, levels=3,
                 host_images=False):
        assert img_wh[0] % 32 == 0 and img_wh[1] % 32 == 0, "img_wh must both be multiples of 32!"
        if split not in self.SCANS or scan not in self.SCANS[split]:
            raise ValueError(f"unknown Tanks and Temples scan {split}/{scan}")
        self.root_dir, self.split, self.scan = root_dir, split, scan
        self.img_wh, self.n_views, self.host_images = tuple(img_wh), n_views, host_images
        self.dir = os.path.join(root_dir, split, scan)
        self.full_wh, self.depth_interval = self.SCANS[split][scan]
        self.metas = io.read_pair_file(os.path.join(self.dir, "pair.txt"))
        self.proj_mats, self.depth_min = _read_proj_mats(
            lambda v: os.path.join(self.dir, "cams", f"{v:08d}_cam.txt"), [r for r, _ in self.metas],
            self.img_wh, self.full_wh, levels)

    def image_path(self, vid):
        return os.path.join(self.dir, "images", f"{vid:08d}.jpg")

    def depth_range(self, ref, depth_interval):
        # torch.FloatTensor([...]).item() of tanks.py:143-144 / eval.py:76-77
        return float(np.float32(self.depth_min[ref])), float(np.float32(self.depth_interval))


class BlendedMVSTestScan(_CachedScan):
    """One BlendedMVS scan in the layout datasets/blendedmvs.py reads (test mode, img_wh given):

        <root>/<scan>/cams/pair.txt, cams/{vid:08d}_cam.txt, blended_images/{vid:08d}.jpg,
        rendered_depth_maps/{vid:08d}.pfm;  scan lists <root>/../{training,validation,all}_list.txt

    Native size 768x576 when root_dir ends in dataset_low_res, else 2048x1536
    (blendedmvs.py:61-65).  Depths are scaled per scan by 100 / depth_min of the first cam
    (:98-103).  Reference views with fewer valid sources than n_views are skipped (:51-54).
    The depth interval of a reference view is
        (max of its rendered depth, scaled and INTER_NEAREST-resized to img_wh, - depth_min) / n_depths_arg
    (:106-126, 170-171), where eval.py passes its --depth_interval as n_depths_arg (eval.py:187-190);
    that is reproduced literally, so the default 2.65 divides the depth range by 2.65."""
    SPLITS = {"train": "training_list.txt", "val": "validation_list.txt", "all": "all_list.txt"}

    def __init__(self, root_dir, scan, img_wh=(768, 576), n_views=5, n_depths_arg=192.0, levels=3,
                 host_images=False):
        assert img_wh[0] % 32 == 0 and img_wh[1] % 32 == 0, "img_wh must both be multiples of 32!"
        self.root_dir, self.scan = root_dir, scan
        self.img_wh, self.n_views, self.host_images = tuple(img_wh), n_views, host_images
        self.dir = os.path.join(root_dir, scan)
        low = root_dir.endswith("dataset_low_res") or root_dir.endswith("dataset_low_res/")
        self.full_wh = (768, 576) if low else (2048, 1536)
        self.metas, refs = [], []
        with open(os.path.join(self.dir, "cams", "pair.txt")) as f:
            for _ in range(int(f.readline())):
                ref = int(f.readline().rstrip())
                refs.append(ref)
                line = f.readline().rstrip().split()
                if int(line[0]) >= n_views:
                    self.metas.append((ref, [int(x) for x in line[1::2]]))
        scale = []
        self.proj_mats, self.depth_min = _read_proj_mats(
            lambda v: os.path.join(self.dir, "cams", f"{v:08d}_cam.txt"), refs, self.img_wh,
            self.full_wh, levels, scale)
        self.scale_factor = scale[0] if scale else None
        self.depth_interval = {}
        for ref, _ in self.metas:
            self.depth_interval[ref] = self._depth_interval(ref, n_depths_arg)

    @staticmethod
    def scans(root_dir, split):
        with open(os.path.join(root_dir, "..", BlendedMVSTestScan.SPLITS[split])) as f:
            return [line.rstrip() for line in f.readlines()]

    def _depth_interval(self, ref, n_depths_arg):
        import cv2
        depth = np.array(io.read_pfm(os.path.join(self.dir, "rendered_depth_maps", f"{ref:08d}.pfm"))[0],
                         dtype=np.float32)
        depth *= self.scale_factor
        depth_max = cv2.resize(depth, self.img_wh, interpolation=cv2.INTER_NEAREST).max()
        return float(np.float32((depth_max - self.depth_min[ref]) / n_depths_arg))

    def image_path(self, vid):
        return os.path.join(self.dir, "blended_images", f"{vid:08d}.jpg")

    def depth_range(self, ref, depth_interval):
        return float(np.float32(self.depth_min[ref])), self.depth_interval[ref]


@torch.no_grad()
def run_scan(model, scan, depth_interval=2.65, conf=0.999, min_geo_consistent=5,
             skip=1, max_ref_views=400, device="cuda:0", depth_dir=None, ply_path=None,
             dtu_gt=None, dtu_seed=0, save_visual=False):
    """-> (xyz (N,3) float32, rgb (N,3) uint8) CUDA tensors; optional PFM / PLY outputs.
    `scan` is a DTUTestScan, TanksTestScan or BlendedMVSTestScan; each gives the depth range of
    its reference views (scan.depth_range).  With `save_visual` and `depth_dir`, the JET depth
    and thresholded confidence JPEGs of eval.py:230-239 are written too.
    With `dtu_gt` (a DTU ground-truth directory) the fused cloud is also scored by
    dtu_eval.evaluate_scan from the device tensors, the scores are written next to the PLY as
    <ply>_scores.json when ply_path is given, and (xyz, rgb, scores) is returned."""
    depths, probas = {}, {}
    writer = io.DepthWriter(depth_dir) if depth_dir else None
    for ref, imgs, pm in scan.views(device):
        dmin, dint = scan.depth_range(ref, depth_interval)
        res = model(imgs.unsqueeze(0), pm.unsqueeze(0).to(device), dmin, dint)
        depths[ref] = torch.nan_to_num(res["depth_0"][0]).clone()            # eval.py:224-227
        probas[ref] = torch.nan_to_num(res["confidence_2"][0]).clone()
        if writer:
            d, p = depths[ref].cpu().numpy(), probas[ref].cpu().numpy()
            writer(scan.scan, ref, d, p)
            if save_visual:
                io.save_visual(depth_dir, scan.scan, ref, d, p, conf)
    images = scan.fusion_images(list(depths), device)
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


def open_scans(a):
    """The scans eval.py:186-196 evaluates, --scan or every scan of the split, opened one at a
    time so that only one scan's image cache is alive."""
    if a.dataset_name == "dtu":
        yield DTUTestScan(a.root_dir, a.scan, tuple(a.img_wh), a.n_views)
        return
    if a.dataset_name == "tanks":
        for s in [a.scan] if a.scan else list(TanksTestScan.SCANS[a.split]):
            yield TanksTestScan(a.root_dir, a.split, s, tuple(a.img_wh), a.n_views)
        return
    for s in [a.scan] if a.scan else BlendedMVSTestScan.scans(a.root_dir, a.split):
        yield BlendedMVSTestScan(a.root_dir, s, tuple(a.img_wh), a.n_views, a.depth_interval)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--root_dir", required=True)
    ap.add_argument("--dataset_name", default="dtu", choices=["dtu", "tanks", "blendedmvs"])
    ap.add_argument("--split", default="test",
                    help="tanks: intermediate | advanced; blendedmvs: train | val | all; dtu: unused")
    ap.add_argument("--scan", default="", help="one scan (default: every scan of the split; dtu needs it)")
    ap.add_argument("--ckpt", default="")
    ap.add_argument("--img_wh", nargs=2, type=int, default=[1152, 864])
    ap.add_argument("--n_views", type=int, default=5)
    ap.add_argument("--n_depths", nargs="+", type=int, default=[8, 32, 48])
    ap.add_argument("--interval_ratios", nargs="+", type=float, default=[1.0, 2.0, 4.0])
    ap.add_argument("--num_groups", type=int, default=1)
    ap.add_argument("--depth_interval", type=float, default=2.65,
                    help="dtu: the depth interval; tanks: no effect; blendedmvs: divides each view's depth range")
    ap.add_argument("--conf", type=float, default=0.999)
    ap.add_argument("--min_geo_consistent", type=int, default=5)
    ap.add_argument("--max_ref_views", type=int, default=400)
    ap.add_argument("--skip", type=int, default=1)
    ap.add_argument("--precision", default="tf32", choices=["fp32", "tf32"])
    ap.add_argument("--save_visual", action="store_true", help="JET depth and confidence-mask JPEGs")
    ap.add_argument("--out", default=None, help="output directory (default results/<dataset_name>)")
    ap.add_argument("--dtu_gt", default=None, help="DTU ground-truth directory: score the fused cloud")
    ap.add_argument("--dtu_seed", type=int, default=0)
    a = ap.parse_args(argv)
    if a.dtu_gt is not None and a.dataset_name != "dtu":
        raise SystemExit("--dtu_gt applies to dtu only")
    if a.dataset_name == "dtu" and not a.scan:
        raise SystemExit("--scan is required for dtu")
    splits = {"tanks": TanksTestScan.SCANS, "blendedmvs": BlendedMVSTestScan.SPLITS}.get(a.dataset_name)
    if splits is not None and a.split not in splits:
        raise SystemExit(f"--split must be one of {sorted(splits)} for {a.dataset_name}")
    out_dir = a.out or os.path.join("results", a.dataset_name)
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
    os.makedirs(os.path.join(out_dir, "points"), exist_ok=True)
    for scan in open_scans(a):
        out = run_scan(model, scan, a.depth_interval, a.conf, a.min_geo_consistent, a.skip,
                       a.max_ref_views, depth_dir=os.path.join(out_dir, "depth"),
                       ply_path=os.path.join(out_dir, "points", f"{scan.scan}.ply"), dtu_gt=a.dtu_gt,
                       dtu_seed=a.dtu_seed, save_visual=a.save_visual)
        print(f"{scan.scan} contains {len(out[0]) / 1e6:.2f} M points")
        if a.dtu_gt is not None:
            from .dtu_eval import _fmt
            print(_fmt(out[2]))


if __name__ == "__main__":
    main()
