"""DTU training reader: datasets/dtu.py of the reference with img_wh=None (train / val).

    <root>/Cameras/pair.txt                      viewpoints and their source views
    <root>/Cameras/train/{vid:08d}_cam.txt       the 49 training cameras (1/4-resolution K)
    <root>/Rectified/<scan>_train/rect_{vid+1:03d}_{light}_r5000.png   640x512, lights 0-6
    <root>/Depths/<scan>/depth_map_{vid:04d}.pfm, depth_visual_{vid:04d}.png   1600x1200

One sample per (scan, light 0-6, viewpoint), sources in pair order.  The reference downsamples
the depth and mask maps with cv2 INTER_NEAREST at 0.5, crops [44:556, 80:720] and halves twice
more.  On even sizes cv2's nearest rule at fx = 0.5 takes source index 2x, so the pyramid is
strided slicing of the full map (tests/golden/train/reader.npz pins the equivalence).

The Dataset runs in DataLoader workers and stays on the host: it decodes the files and returns
the images as uint8 (V,H,W,3).  `to_device` uploads a batch from pinned memory and normalises
the images there (io.normalize_images), giving the reference's sample layout on the GPU.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import io
from .eval_pipeline import read_network_image_u8

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
    normalised on the device, proj_mats, depths / masks {level_l}, init_depth_min and
    depth_interval (B,1)."""
    u8 = batch["imgs_u8"]
    B, V, H, W, _ = u8.shape
    imgs = io.normalize_images(u8.reshape(B * V, H, W, 3).to(device, non_blocking=True))
    mv = lambda d: {k: v.to(device, non_blocking=True) for k, v in d.items()}   # noqa: E731
    return {"imgs": imgs.view(B, V, 3, H, W),
            "proj_mats": batch["proj_mats"].to(device, non_blocking=True),
            "depths": mv(batch["depths"]), "masks": mv(batch["masks"]),
            "init_depth_min": batch["init_depth_min"].to(device, non_blocking=True),
            "depth_interval": batch["depth_interval"].to(device, non_blocking=True),
            "scan_vid": batch["scan_vid"]}
