"""Training readers: datasets/dtu.py of the reference with img_wh=None (DTUTrainDataset) and
datasets/blendedmvs.py in training mode (BlendedMVSTrainDataset), splits train / val.

DTU:

    <root>/Cameras/pair.txt                      viewpoints and their source views
    <root>/Cameras/train/{vid:08d}_cam.txt       the 49 training cameras (1/4-resolution K)
    <root>/Rectified/<scan>_train/rect_{vid+1:03d}_{light}_r5000.png   640x512, lights 0-6
    <root>/Depths/<scan>/depth_map_{vid:04d}.pfm, depth_visual_{vid:04d}.png   1600x1200

One sample per (scan, light 0-6, viewpoint), sources in pair order.  The reference downsamples
the depth and mask maps with cv2 INTER_NEAREST at 0.5, crops [44:556, 80:720] and halves twice
more.  On even sizes cv2's nearest rule at fx = 0.5 takes source index 2x, so the pyramid is
strided slicing of the full map (tests/golden/train/reader.npz pins the equivalence).

BlendedMVS (BlendedMVSTrainDataset; the layout eval_pipeline.BlendedMVSTestScan reads):

    <root>/<scan>/cams/pair.txt, cams/{vid:08d}_cam.txt, blended_images/{vid:08d}.jpg,
    rendered_depth_maps/{vid:08d}.pfm;  scan lists <root>/../{training,validation,all}_list.txt

The training split's images go through T.ColorJitter(brightness=0.25, contrast=0.5) in the
reference.  The worker draws its factors with the torch calls ColorJitter.get_params makes, so
it consumes torch's random numbers exactly as the reference does, and returns them with the
undecorated bytes; the jitter itself runs on the device (io.jitter_normalize_images).

A Dataset runs in DataLoader workers and stays on the host: it decodes the files and returns
the images as uint8 (V,H,W,3).  `to_device` uploads a batch from pinned memory and normalises
the images there (io.normalize_images, or io.jitter_normalize_images when the batch carries
jitter factors), giving the reference's sample layout on the GPU.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import io
from .eval_pipeline import (BlendedMVSTestScan, read_blendedmvs_cams, read_blendedmvs_depth,
                            read_network_image_u8)

N_CAMS = 49
LIGHTS = range(7)
CROP = (slice(44, 556), slice(80, 720))      # of the half-resolution (600, 800) map


def read_scan_list(path):
    """One scan per line (the format of the reference's datasets/lists/dtu/*.txt)."""
    with open(path) as f:
        return [line.strip() for line in f if line.strip()]


def depth_pyramid(full, levels=3):
    """(1200,1600) map -> {level_l: (512/2^l, 640/2^l)}: cv2.resize(fx=fy=0.5, INTER_NEAREST),
    crop, then two more nearest halvings (datasets/dtu.py:92-130)."""
    lvl = np.ascontiguousarray(full[::2, ::2][CROP])
    out = {"level_0": lvl}
    for l in range(1, levels):
        lvl = np.ascontiguousarray(lvl[::2, ::2])
        out[f"level_{l}"] = lvl
    return out


class DTUTrainDataset(torch.utils.data.Dataset):
    """datasets/dtu.py DTUDataset(img_wh=None) over the scans of `scans` (a list)."""

    def __init__(self, root_dir, scans, n_views=3, levels=3, depth_interval=2.65):
        self.root_dir, self.scans = root_dir, list(scans)
        self.n_views, self.levels, self.depth_interval = n_views, levels, depth_interval
        pairs = io.read_pair_file(os.path.join(root_dir, "Cameras", "pair.txt"))
        self.metas = [(scan, light, ref, srcs) for scan in self.scans for ref, srcs in pairs
                      for light in LIGHTS]
        self.proj_mats, self.depth_min = {}, {}
        for vid in range(N_CAMS):
            K, E, dmin = io.read_cam_file(os.path.join(root_dir, "Cameras", "train", f"{vid:08d}_cam.txt"))
            self.proj_mats[vid] = io.pyramid_proj_mats(K, E, levels)
            self.depth_min[vid] = dmin

    def __len__(self):
        return len(self.metas)

    def image_path(self, scan, vid, light):
        return os.path.join(self.root_dir, "Rectified", f"{scan}_train",
                            f"rect_{vid + 1:03d}_{light}_r5000.png")

    def read_depth(self, scan, vid):
        full = np.array(io.read_pfm(os.path.join(self.root_dir, "Depths", scan,
                                                 f"depth_map_{vid:04d}.pfm"))[0], dtype=np.float32)
        return {k: torch.from_numpy(v) for k, v in depth_pyramid(full, self.levels).items()}

    def read_mask(self, scan, vid):
        import cv2
        path = os.path.join(self.root_dir, "Depths", scan, f"depth_visual_{vid:04d}.png")
        full = cv2.imread(path, 0)
        if full is None:
            raise FileNotFoundError(path)
        return {k: torch.from_numpy(v != 0) for k, v in depth_pyramid(full, self.levels).items()}

    def __getitem__(self, idx):
        scan, light, ref, srcs = self.metas[idx]
        ids = [ref] + srcs[: self.n_views - 1]
        imgs = np.stack([read_network_image_u8(self.image_path(scan, v, light), (640, 512)) for v in ids])
        return {"imgs_u8": torch.from_numpy(imgs),
                "proj_mats": io.relative_proj_mats(self.proj_mats, ids),
                "depths": self.read_depth(scan, ref),
                "masks": self.read_mask(scan, ref),
                "init_depth_min": torch.FloatTensor([self.depth_min[ref]]),
                "depth_interval": torch.FloatTensor([self.depth_interval]),
                "scan_vid": (scan, ref)}


BRIGHTNESS = (0.75, 1.25)      # ColorJitter(brightness=0.25) of datasets/blendedmvs.py:132
CONTRAST = (0.5, 1.5)          # ColorJitter(contrast=0.5)


def draw_jitter():
    """One view's ColorJitter(brightness=0.25, contrast=0.5) parameters, drawn from torch's
    global RNG with the calls of ColorJitter.get_params: randperm(4), then a brightness and a
    contrast factor (saturation and hue are unset and draw nothing).  -> (brightness_first, b, c)
    where brightness_first says whether brightness (0) precedes contrast (1) in the order."""
    order = torch.randperm(4).tolist()
    b = float(torch.empty(1).uniform_(*BRIGHTNESS))
    c = float(torch.empty(1).uniform_(*CONTRAST))
    return float(order.index(0) < order.index(1)), b, c


class BlendedMVSTrainDataset(torch.utils.data.Dataset):
    """datasets/blendedmvs.py BlendedMVSDataset(root_dir, split, n_views, levels, n_depths_arg,
    img_wh) in training mode.  Samples are the non-skipped reference views of every scan of the
    split's list, in list and pair order.  Per sample: the views' images PIL-resized to img_wh
    (uint8), the reference view's depths (scaled, INTER_NEAREST to img_wh, halved twice) and
    masks depth_l > depth_min, init_depth_min, and depth_interval =
    (max depth_0 - depth_min) / n_depths_arg; for split 'train' also `jitter` (V,3), one
    draw_jitter() per view in view order."""

    def __init__(self, root_dir, split, n_views=3, levels=3, n_depths_arg=192.0, img_wh=(768, 576)):
        if split not in BlendedMVSTestScan.SPLITS:
            raise ValueError(f"split must be one of {sorted(BlendedMVSTestScan.SPLITS)}, not {split!r}")
        assert img_wh[0] % 32 == 0 and img_wh[1] % 32 == 0, "img_wh must both be multiples of 32!"
        self.root_dir, self.split, self.img_wh = root_dir, split, tuple(img_wh)
        self.n_views, self.levels, self.n_depths_arg = n_views, levels, n_depths_arg
        self.scans = BlendedMVSTestScan.scans(root_dir, split)
        self.metas, self.proj_mats, self.depth_min, self.scale_factors = [], {}, {}, {}
        for scan in self.scans:
            _, metas, self.proj_mats[scan], self.depth_min[scan], self.scale_factors[scan] = \
                read_blendedmvs_cams(root_dir, scan, self.img_wh, n_views, levels)
            self.metas += [(scan, -1, ref, srcs) for ref, srcs in metas]

    def __len__(self):
        return len(self.metas)

    def image_path(self, scan, vid):
        return os.path.join(self.root_dir, scan, "blended_images", f"{vid:08d}.jpg")

    def read_depth_and_mask(self, scan, ref):
        """-> depths, masks {level_l}, depth_max (datasets/blendedmvs.py:106-128)."""
        import cv2
        depth_min = self.depth_min[scan][ref]
        lvl = read_blendedmvs_depth(os.path.join(self.root_dir, scan), ref, self.scale_factors[scan],
                                    self.img_wh)
        depths, masks = {}, {}
        for l in range(self.levels):
            if l:
                lvl = cv2.resize(lvl, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_NEAREST)
            depths[f"level_{l}"] = torch.from_numpy(np.ascontiguousarray(lvl))
            masks[f"level_{l}"] = torch.from_numpy(lvl > depth_min)
        return depths, masks, depths["level_0"].numpy().max()

    def __getitem__(self, idx):
        scan, _, ref, srcs = self.metas[idx]
        ids = [ref] + srcs[: self.n_views - 1]
        imgs, jitter = [], []
        for vid in ids:                      # the reference decodes, then transforms, per view
            imgs.append(read_network_image_u8(self.image_path(scan, vid), self.img_wh))
            if self.split == "train":
                jitter.append(draw_jitter())
        depth_min = self.depth_min[scan][ref]
        depths, masks, depth_max = self.read_depth_and_mask(scan, ref)
        sample = {"imgs_u8": torch.from_numpy(np.stack(imgs)),
                  "proj_mats": io.relative_proj_mats(self.proj_mats[scan], ids),
                  "depths": depths, "masks": masks,
                  "init_depth_min": torch.FloatTensor([depth_min]),
                  "depth_interval": torch.FloatTensor([(depth_max - depth_min) / self.n_depths_arg]),
                  "scan_vid": (scan, ref)}
        if jitter:
            sample["jitter"] = torch.tensor(jitter, dtype=torch.float32)
        return sample


def loader(dataset, batch_size, shuffle, num_workers=4, seed=None):
    """Host-only workers (decode and slice), pinned batches."""
    g = None
    if seed is not None:
        g = torch.Generator()
        g.manual_seed(seed)
    return torch.utils.data.DataLoader(dataset, batch_size=batch_size, shuffle=shuffle,
                                       num_workers=num_workers, pin_memory=True, generator=g,
                                       persistent_workers=num_workers > 0)


def to_device(batch, device):
    """A collated host batch -> the reference's sample dict on `device`: imgs (B,V,3,H,W)
    normalised on the device (after the colour jitter when the batch carries `jitter`), proj_mats, depths / masks {level_l}, init_depth_min and
    depth_interval (B,1)."""
    u8 = batch["imgs_u8"]
    B, V, H, W, _ = u8.shape
    u8 = u8.reshape(B * V, H, W, 3).to(device, non_blocking=True)
    if "jitter" in batch:
        imgs = io.jitter_normalize_images(u8, batch["jitter"].reshape(B * V, 3).to(device, non_blocking=True))
    else:
        imgs = io.normalize_images(u8)
    mv = lambda d: {k: v.to(device, non_blocking=True) for k, v in d.items()}   # noqa: E731
    return {"imgs": imgs.view(B, V, 3, H, W),
            "proj_mats": batch["proj_mats"].to(device, non_blocking=True),
            "depths": mv(batch["depths"]), "masks": mv(batch["masks"]),
            "init_depth_min": batch["init_depth_min"].to(device, non_blocking=True),
            "depth_interval": batch["depth_interval"].to(device, non_blocking=True),
            "scan_vid": batch["scan_vid"]}
