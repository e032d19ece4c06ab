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

and over a scene of the user's own, reconstructed by COLMAP:

    colmap      ColmapScan          <root>/images (or --image_dir), <root>/sparse[/0]/{cameras,
                                    images,points3D}.{bin,txt}; view selection and depth ranges
                                    computed here (colmap.py); views of a distorted camera are
                                    undistorted on the GPU as they are read (io.undistort_u8)

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
    python -m casmvsnet_pl_b200.eval_pipeline --dataset_name colmap --root_dir my_capture/dense \
        --ckpt ckpt.ckpt --img_wh 1152 864 [--depth_interval 192] [--mesh [--mesh_voxel S]]
    python -m casmvsnet_pl_b200.eval_pipeline --dataset_name colmap --root_dir my_capture \
        --image_dir my_capture/photos --ckpt ckpt.ckpt     (a `colmap mapper` project, sparse/0)

--mesh also fuses each scan's filtered depth maps into a TSDF volume on the GPU and writes the
marching-cubes mesh to <out>/mesh/<scan>.ply (mesh.py); nothing else it writes changes.
--mesh --mesh_method poisson [--poisson_depth 9] meshes the scan's fused points by Poisson surface
reconstruction instead (poisson.py); --poisson_point_weight A > 0 screens it.
--mesh --mesh_clean drops either mesh's small disconnected pieces (--mesh_clean_ratio R of the
largest piece's faces, default 0.01) and fills its holes of at most --mesh_max_hole E edges
(default 0: none) on the GPU before anything else sees it (mesh_clean.py).
--mesh --mesh_faces N decimates either mesh to at most N faces on the GPU before it is written
(simplify.py).
--mesh --mesh_texture also textures the mesh that is written from the scan's reference-view images
at --img_wh and writes <out>/mesh/<scan>.obj, .mtl and _<k>.png beside the PLY (texture.py);
--mesh_texture_level also levels the colour seams between its charts, changing only the PNGs.
--mesh --mesh_score with --dtu_gt or --tnt_gt also scores the mesh as it is written, through its
surface samples (dtu_eval.evaluate_mesh / tnt_eval.evaluate_mesh), into <out>/mesh/<scan>_scores.json
or <out>/mesh/<scan>_tnt.json.
--remove_outliers [--outlier_neighbours K] [--outlier_std R] removes the fused cloud's statistical
outliers on the GPU (cloud_filter.py) before it is written, scored or Poisson-meshed.
"""
from __future__ import annotations

import argparse
import json
import math
import os

import numpy as np
import torch

from . import fusion, io

# --num_groups values (eval_pipeline and train.py): the group-wise correlation splits the
# 8 / 16 / 32 feature channels of every stage into this many groups
NUM_GROUPS = (1, 2, 4, 8)


def depth_count(text):
    """argparse type of --n_depths: CostRegNet halves the depth three times and back, so each
    stage's plane count must be a positive multiple of 8."""
    n = int(text)
    if n <= 0 or n % 8:
        raise argparse.ArgumentTypeError(f"{text} is not a positive multiple of 8")
    return n


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
    is decoded once instead of once per reference view it takes part in, plus once for fusion.
    `cameras` {view: (src_cam, dst_cam)} (io.undistort_u8's camera pair) names the views of a
    distorted camera: both decodes of such a view must be the camera's size, and are undistorted
    to its pinhole camera in one call before they are resized."""

    def __init__(self, paths, img_wh, device, workers=4, cameras=None):
        from concurrent.futures import ThreadPoolExecutor
        self.index = {v: i for i, v in enumerate(paths)}
        cameras = cameras or {}
        w, h = img_wh
        n = len(self.index)
        self.net = torch.empty(n, h, w, 3, dtype=torch.uint8, device=device)
        self.fus = torch.empty(n, h, w, 3, dtype=torch.uint8, device=device)
        with ThreadPoolExecutor(max(1, workers)) as ex:
            for i, (v, (pil, bgr)) in enumerate(zip(paths, ex.map(_decode_pil_cv2, paths.values()))):
                if v in cameras:
                    src, dst = cameras[v]
                    for img in (pil, bgr):
                        if img.shape[:2] != (src[2], src[1]):
                            raise ValueError(f"{paths[v]}: the image is {img.shape[1]}x{img.shape[0]}, "
                                             f"its camera {src[1]}x{src[2]}")
                    both = torch.from_numpy(np.stack([pil, bgr])).pin_memory()
                    und = io.undistort_u8(both.to(device, non_blocking=True), src, dst)
                    io.resize_u8_pil(und[0:1], img_wh, out=self.net[i:i + 1])
                    io.resize_u8_linear(und[1:2], img_wh, out=self.fus[i:i + 1])
                    continue
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
    camera_pairs = None          # SceneImages' `cameras`: views to undistort
    _images = None

    def _image_cache(self, device):
        if self._images is None:
            self._images = SceneImages({v: self.image_path(v) for v in self.proj_mats}, self.img_wh,
                                       device, cameras=self.camera_pairs)
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


def read_blendedmvs_cams(root_dir, scan, img_wh, n_views, levels):
    """build_metas + build_proj_mats of datasets/blendedmvs.py:32-104 for one scan ->
    (full_wh, metas [(ref, srcs)], proj_mats {vid}, depth_min {vid}, scale_factor).  The native
    size is 768x576 when root_dir ends in dataset_low_res, else 2048x1536 (:61-65); reference
    views with fewer valid sources than n_views are left out of metas (:51-54), but every view
    of pair.txt gets its projections; depth_min and the extrinsic translation are scaled by
    100 / depth_min of the first cam read (:98-103)."""
    d = os.path.join(root_dir, scan)
    low = root_dir.endswith("dataset_low_res") or root_dir.endswith("dataset_low_res/")
    full_wh = (768, 576) if low else (2048, 1536)
    metas, refs = [], []
    with open(os.path.join(d, "cams", "pair.txt")) as f:
        for _ in range(int(f.readline())):
            ref = int(f.readline().rstrip())
            refs.append(ref)
            line = f.readline().rstrip().split()
            if int(line[0]) >= n_views:
                metas.append((ref, [int(x) for x in line[1::2]]))
    scale = []
    proj_mats, depth_min = _read_proj_mats(lambda v: os.path.join(d, "cams", f"{v:08d}_cam.txt"),
                                           refs, img_wh, full_wh, levels, scale)
    return full_wh, metas, proj_mats, depth_min, (scale[0] if scale else None)


def read_blendedmvs_depth(scan_dir, vid, scale_factor, img_wh):
    """A view's rendered depth, scaled by the scan's factor and cv2 INTER_NEAREST-resized to
    img_wh (datasets/blendedmvs.py:106-111) -> (h,w) float32."""
    import cv2
    depth = np.array(io.read_pfm(os.path.join(scan_dir, "rendered_depth_maps", f"{vid:08d}.pfm"))[0],
                     dtype=np.float32)
    depth *= scale_factor
    return cv2.resize(depth, tuple(img_wh), interpolation=cv2.INTER_NEAREST)


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
        self.full_wh, self.metas, self.proj_mats, self.depth_min, self.scale_factor = \
            read_blendedmvs_cams(root_dir, scan, self.img_wh, n_views, levels)
        self.depth_interval = {}
        for ref, _ in self.metas:
            self.depth_interval[ref] = self._depth_interval(ref, n_depths_arg)

    @staticmethod
    def scans(root_dir, split):
        with open(os.path.join(root_dir, "..", BlendedMVSTestScan.SPLITS[split])) as f:
            return [line.rstrip() for line in f.readlines()]

    def _depth_interval(self, ref, n_depths_arg):
        depth_max = read_blendedmvs_depth(self.dir, ref, self.scale_factor, self.img_wh).max()
        return float(np.float32((depth_max - self.depth_min[ref]) / n_depths_arg))

    def image_path(self, vid):
        return os.path.join(self.dir, "blended_images", f"{vid:08d}.jpg")

    def depth_range(self, ref, depth_interval):
        return float(np.float32(self.depth_min[ref])), self.depth_interval[ref]


class ColmapScan(_CachedScan):
    """A scene reconstructed by COLMAP, in the workspace `colmap image_undistorter` writes or as
    a `colmap mapper` project:

        <image_dir>/<name> (default <root>/images),
        <root>/sparse/{cameras,images,points3D}.{bin,txt} (or <root>/sparse/0/...)

    A view of a distorted camera (colmap.DISTORTED_MODELS) is computed in its undistorted
    PINHOLE camera (colmap.undistorted_camera): K, the projections and the written cams are that
    camera's, and its images are undistorted on the GPU as SceneImages reads them.  The host
    route (host_images=True) has no undistortion and refuses such a scene.

    Views are numbered 0..n-1 in sorted image-name order.  Each view's sources are the N_SRC
    views with the best positive view-selection score (colmap.py; the scores are computed on the
    GPU by casmvs_view_scores_fwd).  A view is not a reference view when it has fewer than
    n_views - 1 sources or fewer than 20 observed points in front of it; `skipped` maps those to
    the reason.  A reference view's depth range is [0.75 q(0.01), 1.25 q(0.99)] of the depths of
    its observed points and its depth interval that range / n_depths_arg.  Intrinsics are the
    full-resolution K of the view's (undistorted) camera, scaled to img_wh like Tanks'.
    With `out_dir`, the run is recorded in <out_dir>/<scan>: cams/{vid:08d}_cam.txt for every
    view (MVSNet format: extrinsic, full-resolution intrinsic, `depth_min interval n_depths
    depth_max`, nan for a view with no point in front of it), pair.txt with the reference views
    and their scored sources, and view_names.txt (view id -> image name)."""

    def __init__(self, root_dir, scan=None, img_wh=(1152, 864), n_views=5, n_depths_arg=192.0,
                 levels=3, host_images=False, out_dir=None, device="cuda:0", log=print,
                 image_dir=None):
        from . import colmap
        assert img_wh[0] % 32 == 0 and img_wh[1] % 32 == 0, "img_wh must both be multiples of 32!"
        self.root_dir = root_dir
        self.image_dir = image_dir or os.path.join(root_dir, "images")
        self.scan = scan or os.path.basename(os.path.normpath(os.path.abspath(root_dir)))
        self.img_wh, self.n_views, self.host_images = tuple(img_wh), n_views, host_images
        sc = self.scene = colmap.load_scene(root_dir)
        if len(sc) == 0:
            raise ValueError(f"{root_dir}: the COLMAP model has no registered images")
        if sc.distorted.any():
            if host_images:
                v = int(np.argmax(sc.distorted))
                raise ValueError(f"{root_dir}: view {v} ({sc.names[v]}) has a distorted camera "
                                 f"({colmap.CAMERA_MODELS[sc.src_cameras[v][0]][0]}); the host "
                                 "image route (host_images=True) has no undistortion")
            self.camera_pairs = {
                int(v): (sc.src_cameras[v], (int(sc.wh[v, 0]), int(sc.wh[v, 1]),
                                             sc.K[v][[0, 1, 0, 1], [0, 1, 2, 2]]))
                for v in np.nonzero(sc.distorted)[0]}
        scores = colmap.view_scores(sc.centres, sc.xyz, sc.track_ptr, sc.track_img, device)
        count, q = colmap.depth_stats(sc.E, sc.xyz, sc.track_ptr, sc.track_img, device)
        self.scores = scores.cpu().numpy()
        sources, refs, self.skipped, dmin, dmax = colmap.assemble(self.scores, count, q, n_views)
        self.metas = [(r, [s for s, _ in sources[r]]) for r in refs]
        E32, K32 = sc.E.astype(np.float32), sc.K.astype(np.float32)
        self.proj_mats = {v: io.pyramid_proj_mats(K32[v], E32[v], levels, self.img_wh,
                                                  tuple(int(x) for x in sc.wh[v]))
                          for v in range(len(sc))}
        self.depth_min, self.depth_interval, self.depth_max = {}, {}, {}
        for v in range(len(sc)):            # NaN for a view with no point in front of it
            self.depth_min[v] = float(np.float32(dmin[v]))
            self.depth_interval[v] = float(np.float32((dmax[v] - dmin[v]) / n_depths_arg))
            self.depth_max[v] = float(dmax[v])
        for v, why in sorted(self.skipped.items()):
            log(f"{self.scan}: view {v} ({sc.names[v]}) is not a reference view: {why}")
        if out_dir:
            d = os.path.join(out_dir, self.scan)
            os.makedirs(d, exist_ok=True)
            colmap.write_cams(os.path.join(d, "cams"), E32, K32,
                              {v: (self.depth_min[v], self.depth_interval[v], self.depth_max[v])
                               for v in range(len(sc))}, n_depths_arg)
            colmap.write_pair(os.path.join(d, "pair.txt"), [(r, sources[r]) for r in refs])
            colmap.write_view_names(os.path.join(d, "view_names.txt"), sc.names)

    def image_path(self, vid):
        return os.path.join(self.image_dir, self.scene.names[vid])

    def depth_range(self, ref, depth_interval):
        # the divisor was applied at construction (n_depths_arg)
        return self.depth_min[ref], self.depth_interval[ref]


def _simplify(name, verts, colours, faces, mesh_faces, log):
    """The mesh decimated to `mesh_faces` faces (unchanged when it is None)."""
    if mesh_faces is None:
        return verts, colours, faces
    from . import simplify
    verts, colours, faces, st = simplify.simplify_mesh(verts, colours, faces, mesh_faces, log=log)
    log(f"{name}: simplified the mesh from {st['faces_in']} to {st['faces']} faces in "
        f"{st['rounds']} rounds")
    return verts, colours, faces


def _remove_outliers(name, xyz, outlier_filter, log):
    """-> (the points cloud_filter.filter_points keeps, their indices), or (xyz, None) for a
    cloud of k points or fewer, which is kept whole."""
    from . import cloud_filter
    k = outlier_filter.get("k", cloud_filter.DEFAULT_K)
    std_ratio = outlier_filter.get("std_ratio", cloud_filter.DEFAULT_STD_RATIO)
    if len(xyz) <= k:
        log(f"{name}: outliers not removed: {len(xyz)} points, and the filter needs more than "
            f"k = {k}")
        return xyz, None
    kept, index, st = cloud_filter.filter_points(xyz, k, std_ratio)
    log(f"{name}: removed outliers: {cloud_filter.summary(st)}")
    return kept, index


def _clean(name, verts, colours, faces, mesh_clean, log):
    """The mesh cleaned by mesh_clean.clean_mesh(**mesh_clean) (unchanged when it is None)."""
    if mesh_clean is None:
        return verts, colours, faces
    from . import mesh_clean as mc
    verts, colours, faces, st = mc.clean_mesh(verts, colours, faces, **mesh_clean)
    log(f"{name}: cleaned the mesh: {mc.summary(st)}")
    return verts, colours, faces


def _refine(name, verts, colours, faces, images, proj0, metas, iterations, log):
    """The mesh refined against the reference views' images (cast to uint8), proj0 and the scan's
    pair sources by refine.refine_mesh (unchanged when iterations is None)."""
    if iterations is None:
        return verts, colours, faces
    from . import refine
    vids = sorted(images)
    ims = [images[v].to(torch.uint8).contiguous() for v in vids]
    sources = refine.pair_sources(metas, vids)
    verts, colours, faces, st = refine.refine_mesh(verts, colours, faces, ims, [proj0[v] for v in vids],
                                                   sources, iterations=iterations, log=log)
    log(f"{name}: refined the mesh against {st['views']} views: {refine.summary(st)}")
    return verts, colours, faces


def _score_mesh(scan, mesh_path, verts, faces, dtu_gt, dtu_seed, tnt_gt, tnt_images, tnt_tau,
                tnt_seed, run_dir):
    """Scores of the written mesh against the Tanks and Temples (tnt_gt) or DTU (dtu_gt) ground
    truth, written beside it as <mesh>_tnt.json or <mesh>_scores.json."""
    stem = os.path.splitext(mesh_path)[0]
    if tnt_gt is not None:
        from . import tnt_eval
        scores = tnt_eval.evaluate_mesh((verts, faces), run_dir, tnt_gt, scan.scan, tnt_tau, tnt_seed,
                                        images=tnt_images)
        tnt_eval.write_json(stem + "_tnt.json", scores)
        return scores
    from . import dtu_eval
    scores = dtu_eval.evaluate_mesh((verts, faces), dtu_eval.scan_number(scan.scan), dtu_gt,
                                    seed=dtu_seed)
    with open(stem + "_scores.json", "w") as f:
        json.dump(scores, f, indent=1)
    return scores


def _texture(name, mesh_path, verts, colours, faces, images, proj0, log, level=False):
    """Texture the written mesh from the reference views' images (cast to uint8) and proj0, and
    write <mesh_path without .ply>.obj / .mtl / _<k>.png; with `level`, the seams are levelled."""
    from . import texture
    vids = sorted(images)
    ims = [images[v].to(torch.uint8).contiguous() for v in vids]
    uv, page, atlas, st = texture.texture_mesh(verts, colours, faces, ims, [proj0[v] for v in vids],
                                               level=level, log=log)
    texture.write_textured_obj(os.path.splitext(mesh_path)[0] + ".obj", verts, faces, uv, page, atlas)
    log(f"{name}: textured {st['faces']} faces from {st['views']} views: {st['unseen_faces']} "
        f"unseen, {st['charts']} charts on {st['pages']} pages ({st['packed_share']:.1%} packed)")
    if level:
        lv = st["level"]
        log(f"{name}: levelled {lv['seam_pairs']} seam pairs in {lv['cg_iterations']} CG iterations: "
            f"seam RMS {lv['seam_rms_before']:.3f} -> {lv['seam_rms_after']:.3f}")


@torch.no_grad()
def run_scan(model, scan, depth_interval=2.65, conf=0.999, min_geo_consistent=5,
             skip=1, max_ref_views=400, device="cuda:0", depth_dir=None, ply_path=None,
             dtu_gt=None, dtu_seed=0, save_visual=False, mesh_path=None, mesh_voxel=None, log=print,
             tnt_gt=None, tnt_images=None, tnt_tau=None, tnt_seed=0, run_dir=None,
             mesh_method="tsdf", poisson_depth=None, poisson_point_weight=0.0, mesh_faces=None,
             mesh_texture=False, mesh_score=False, mesh_texture_level=False, mesh_clean=None,
             fusion_rule="reference", outlier_filter=None, mesh_refine=None):
    """-> (xyz (N,3) float32, rgb (N,3) uint8) CUDA tensors; optional PFM / PLY outputs.
    `scan` is a DTUTestScan, TanksTestScan, BlendedMVSTestScan or ColmapScan; each gives the depth range of
    its reference views (scan.depth_range).  With `save_visual` and `depth_dir`, the JET depth
    and thresholded confidence JPEGs of eval.py:230-239 are written too.
    With `dtu_gt` (a DTU ground-truth directory) the fused cloud is also scored by
    dtu_eval.evaluate_scan from the device tensors, the scores are written next to the PLY as
    <ply>_scores.json when ply_path is given, and (xyz, rgb, scores) is returned.
    With `mesh_path`, the masked refined depth maps are also fused into a TSDF volume and the
    marching-cubes mesh is written there as a PLY (mesh.py; voxel size `mesh_voxel`, default
    mesh.default_voxel_size); the other outputs are unchanged.  With mesh_method="poisson" the
    mesh is instead the Poisson surface (poisson.py, grid depth `poisson_depth`, default 9) of
    every fused point (not thinned by `skip`), coloured by the refined image at its pixel, its
    normals oriented toward the reference cameras, screened with point weight
    `poisson_point_weight` when it is > 0.  With `mesh_clean` (a dict of mesh_clean.clean_mesh's
    options, possibly empty), either mesh is first cleaned (mesh_clean.py), so that everything
    below sees the cleaned mesh.  With `mesh_faces`, either mesh is decimated to at most
    that many faces (simplify.py) before it is written.  With `mesh_texture`, the written mesh is
    also textured from the reference views' images and proj0 (texture.py) and written beside it
    as an OBJ with its MTL and atlas PNGs; `mesh_texture_level` also levels its colour seams.
    With `mesh_refine` (a number of iterations >= 1), either mesh is refined against the reference
    views' images, proj0 and the scan's pair sources (refine.py) after it is cleaned and
    simplified, before it is written, textured or scored; only its vertices move.
    With `tnt_gt` (a Tanks and Temples ground-truth directory holding the scan's scene) the fused
    cloud is scored by tnt_eval.evaluate_scene from the device tensors against the cameras the run
    recorded in `run_dir`, the scores are written next to the PLY as <ply>_tnt.json when ply_path
    is given, and (xyz, rgb, scores) is returned.
    `fusion_rule` is fusion.fuse_scan's `rule`: "dynamic" fuses with the dynamic consistency
    check (min_geo_consistent is then ignored) and logs the count of kept points; everything
    downstream takes its cloud unchanged.
    With `outlier_filter` (dict(k=..., std_ratio=...), either may be left out for its default),
    the fused cloud (after `skip`) loses its statistical outliers (cloud_filter.py) before it is
    written, scored or returned, and Poisson meshing's unthinned points lose theirs by the same
    rule on that cloud; TSDF meshing is unchanged.  A cloud of k points or fewer is kept whole,
    and the log says so.
    With `mesh_score` (it needs `mesh_path` and `tnt_gt` or `dtu_gt`), the mesh as written is also
    scored through its surface samples by tnt_eval.evaluate_mesh or dtu_eval.evaluate_mesh, the
    scores are written beside it as <mesh>_tnt.json or <mesh>_scores.json, and appended to the
    returned tuple."""
    if mesh_score and (mesh_path is None or (tnt_gt is None and dtu_gt is None)):
        raise ValueError("mesh_score needs mesh_path and a ground truth (dtu_gt or tnt_gt)")
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
    fused = [] if mesh_path else None
    xyz, rgb = fusion.fuse_scan(scan.metas, depths, probas, images, proj0, conf, min_geo_consistent,
                                skip, max_ref_views, collect=fused, rule=fusion_rule)
    if fusion_rule != "reference":
        log(f"{scan.scan}: {fusion_rule} fusion kept {len(xyz)} points")
    kept_index = None
    if outlier_filter is not None:
        xyz, kept_index = _remove_outliers(scan.scan, xyz, outlier_filter, log)
        if kept_index is not None:
            rgb = rgb[kept_index]
    if ply_path:
        fusion.write_ply(ply_path, xyz, rgb)
    if mesh_path and mesh_method == "poisson":
        from . import mesh, poisson
        if not fused:
            raise ValueError(f"{scan.scan}: no reference view was fused, nothing to mesh")
        pts = torch.cat([f["points"] for f in fused]).float()
        cols = torch.cat([f["image"][f["depth"] != 0] for f in fused]).to(torch.uint8)
        if len(cols) != len(pts):
            raise ValueError(f"{scan.scan}: the fused depth maps and points disagree")
        if outlier_filter is not None:
            if skip != 1:                       # Poisson's points are not the written cloud
                _, kept_index = _remove_outliers(f"{scan.scan} (poisson points)", pts,
                                                 outlier_filter, log)
            if kept_index is not None:
                pts, cols = pts[kept_index].contiguous(), cols[kept_index].contiguous()
        cams = np.stack([-np.linalg.inv(np.asarray(f["P"], np.float64)[:3, :3]) @
                         np.asarray(f["P"], np.float64)[:3, 3] for f in fused])
        del fused
        verts, colours, faces, st = poisson.poisson_mesh(
            pts, cols, cam_centres=cams,
            depth=poisson.DEFAULT_DEPTH if poisson_depth is None else poisson_depth, log=log,
            point_weight=poisson_point_weight)
        del pts, cols
        verts, colours, faces = _clean(scan.scan, verts, colours, faces, mesh_clean, log)
        verts, colours, faces = _simplify(scan.scan, verts, colours, faces, mesh_faces, log)
        verts, colours, faces = _refine(scan.scan, verts, colours, faces, images, proj0, scan.metas,
                                        mesh_refine, log)
        mesh.write_mesh_ply(mesh_path, verts, colours, faces)
        if mesh_texture:
            _texture(scan.scan, mesh_path, verts, colours, faces, images, proj0, log,
                     mesh_texture_level)
        written = (verts, faces)
        log(f"{scan.scan}: poisson mesh at depth {st['depth']} (h {st['h']:.6g}): {st['points']} "
            f"points ({st['dropped']} dropped), {st['cycles']} cycles, {st['bricks']} bricks, "
            f"{st['vertices']} vertices, {st['triangles']} triangles")
    elif mesh_path:
        from . import mesh
        if not fused:
            raise ValueError(f"{scan.scan}: no reference view was fused, nothing to mesh")
        verts, colours, faces, st = mesh.mesh_views([f["points"] for f in fused],
                                                    [f["depth"] for f in fused],
                                                    [f["image"] for f in fused],
                                                    [f["P"] for f in fused], mesh_voxel)
        del fused
        verts, colours, faces = _clean(scan.scan, verts, colours, faces, mesh_clean, log)
        verts, colours, faces = _simplify(scan.scan, verts, colours, faces, mesh_faces, log)
        verts, colours, faces = _refine(scan.scan, verts, colours, faces, images, proj0, scan.metas,
                                        mesh_refine, log)
        mesh.write_mesh_ply(mesh_path, verts, colours, faces)
        if mesh_texture:
            _texture(scan.scan, mesh_path, verts, colours, faces, images, proj0, log,
                     mesh_texture_level)
        written = (verts, faces)
        log(f"{scan.scan}: mesh at voxel {st['voxel']:.6g}: {st['bricks']} bricks, {st['voxels']} "
            f"voxels, {st['vertices']} vertices, {st['triangles']} triangles, {st['dropped']} "
            "points dropped")
    extra = ()
    if mesh_score:
        extra = (_score_mesh(scan, mesh_path, *written, dtu_gt, dtu_seed, tnt_gt, tnt_images, tnt_tau,
                             tnt_seed, run_dir),)
    if tnt_gt is not None:
        from . import tnt_eval
        scores = tnt_eval.evaluate_scene(xyz, run_dir, tnt_gt, scan.scan, tnt_tau, tnt_seed,
                                         images=tnt_images)
        if ply_path:
            tnt_eval.write_json(os.path.splitext(ply_path)[0] + "_tnt.json", scores)
        return (xyz, rgb, scores) + extra
    if dtu_gt is None:
        return xyz, rgb
    from . import dtu_eval
    scores = dtu_eval.evaluate_scan(xyz, dtu_eval.scan_number(scan.scan), dtu_gt, seed=dtu_seed)
    if ply_path:
        with open(os.path.splitext(ply_path)[0] + "_scores.json", "w") as f:
            json.dump(scores, f, indent=1)
    return (xyz, rgb, scores) + extra


def open_scans(a):
    """The scans eval.py:186-196 evaluates, --scan or every scan of the split, opened one at a
    time so that only one scan's image cache is alive."""
    if a.dataset_name == "dtu":
        yield DTUTestScan(a.root_dir, a.scan, tuple(a.img_wh), a.n_views)
        return
    if a.dataset_name == "colmap":
        yield ColmapScan(a.root_dir, a.scan or None, tuple(a.img_wh), a.n_views, a.depth_interval,
                         out_dir=a.out_dir, image_dir=a.image_dir)
        return
    if a.dataset_name == "tanks":
        for s in [a.scan] if a.scan else list(TanksTestScan.SCANS[a.split]):
            yield TanksTestScan(a.root_dir, a.split, s, tuple(a.img_wh), a.n_views)
        return
    for s in [a.scan] if a.scan else BlendedMVSTestScan.scans(a.root_dir, a.split):
        yield BlendedMVSTestScan(a.root_dir, s, tuple(a.img_wh), a.n_views, a.depth_interval)


def load_checkpoint(model, path):
    """Weights of a Lightning checkpoint ('model.'-prefixed keys under 'state_dict', as the
    reference's train.py and casmvsnet_pl_b200.train write) or of a plain state dict."""
    sd = torch.load(path, map_location="cpu")
    sd = sd.get("state_dict", sd)
    sd = {k[len("model."):] if k.startswith("model.") else k: v for k, v in sd.items()}   # utils:57-59
    model.load_state_dict(sd)
    return model


DEFAULT_DEPTH_INTERVAL = {"dtu": 2.65, "tanks": 2.65, "blendedmvs": 2.65, "colmap": 192.0}


def parse_args(argv=None):
    """The command line, with --depth_interval resolved per data set (DEFAULT_DEPTH_INTERVAL:
    2.65 as eval.py has it for dtu, tanks and blendedmvs; 192 = 48 x 4 for colmap, so that the
    coarsest stage's 48 planes at interval ratio 4 span a view's depth range exactly) and the
    output directory (default results/<dataset_name>) in `out_dir`."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--root_dir", required=True)
    ap.add_argument("--dataset_name", default="dtu", choices=["dtu", "tanks", "blendedmvs", "colmap"])
    ap.add_argument("--split", default="test",
                    help="tanks: intermediate | advanced; blendedmvs: train | val | all; "
                         "dtu, colmap: unused")
    ap.add_argument("--scan", default="", help="one scan (default: every scan of the split; dtu "
                                               "needs it; colmap: the name of the root directory)")
    ap.add_argument("--image_dir", default=None,
                    help="colmap: the directory holding the model's images (default <root_dir>/images)")
    ap.add_argument("--ckpt", default="")
    ap.add_argument("--img_wh", nargs=2, type=int, default=[1152, 864])
    ap.add_argument("--n_views", type=int, default=5)
    ap.add_argument("--n_depths", nargs="+", type=depth_count, default=[8, 32, 48])
    ap.add_argument("--interval_ratios", nargs="+", type=float, default=[1.0, 2.0, 4.0])
    ap.add_argument("--num_groups", type=int, default=1, choices=NUM_GROUPS)
    ap.add_argument("--depth_interval", type=float, default=None,
                    help="dtu: the depth interval (default 2.65); tanks: no effect; blendedmvs: "
                         "divides each view's depth range (default 2.65); colmap: the same "
                         "(default 192)")
    ap.add_argument("--conf", type=float, default=0.999)
    ap.add_argument("--min_geo_consistent", type=int, default=5)
    ap.add_argument("--fusion", choices=list(fusion.RULES), default=argparse.SUPPRESS,
                    help="the geometric consistency rule: reference (default; at least "
                         "--min_geo_consistent sources within 1 px and 1 %% depth) or dynamic "
                         "(for some k in 2..10, at least k sources within k/4 px and k/1300 "
                         "relative depth)")
    ap.add_argument("--depth_sampling", choices=["uniform", "inverse", "adaptive"],
                    default=argparse.SUPPRESS,
                    help="plane spacing of the sweep: uniform (default; evenly in depth), inverse "
                         "(evenly in 1/depth and regressed in 1/depth, for wide depth ranges) or "
                         "adaptive (each finer stage searches +-1.5 spreads of the previous stage's "
                         "probability volume, at least +-its uniform step)")
    ap.add_argument("--max_ref_views", type=int, default=400)
    ap.add_argument("--skip", type=int, default=1)
    ap.add_argument("--precision", default="tf32", choices=["fp32", "tf32"])
    ap.add_argument("--save_visual", action="store_true", help="JET depth and confidence-mask JPEGs")
    ap.add_argument("--out", default=None, help="output directory (default results/<dataset_name>)")
    ap.add_argument("--dtu_gt", default=None, help="DTU ground-truth directory: score the fused cloud")
    ap.add_argument("--dtu_seed", type=int, default=0)
    ap.add_argument("--tnt_gt", default=None,
                    help="colmap: Tanks and Temples ground-truth directory holding <gt>/<scan>/: "
                         "score the fused cloud (points/<scan>_tnt.json)")
    ap.add_argument("--tnt_images", default=None,
                    help="with --tnt_gt: the complete image directory, to pair cameras by name")
    ap.add_argument("--tnt_tau", type=float, default=None,
                    help="with --tnt_gt: tau for a scene outside the seven training scenes")
    ap.add_argument("--tnt_seed", type=int, default=0)
    ap.add_argument("--mesh", action="store_true",
                    help="also write a TSDF / marching-cubes mesh of each scan to <out>/mesh/<scan>.ply")
    ap.add_argument("--mesh_voxel", type=float, default=None,
                    help="voxel size of --mesh in world units (default: 2 x the median pixel "
                         "footprint at the views' median depth)")
    ap.add_argument("--mesh_method", default=None, choices=["tsdf", "poisson"],
                    help="with --mesh: tsdf (default) fuses the depth maps into a TSDF volume; "
                         "poisson meshes the fused points by Poisson surface reconstruction")
    ap.add_argument("--poisson_depth", type=int, default=None,
                    help="with --mesh_method poisson: the grid depth, 6..10 (default 9)")
    ap.add_argument("--poisson_point_weight", type=float, default=None,
                    help="with --mesh_method poisson: the screening weight alpha >= 0 that pulls "
                         "the surface through the points (default 0, unscreened)")
    ap.add_argument("--mesh_clean", action="store_true",
                    help="with --mesh: drop the mesh's small disconnected pieces (and, with "
                         "--mesh_max_hole, fill its small holes) on the GPU before it is "
                         "simplified, textured, scored or written")
    ap.add_argument("--mesh_clean_ratio", type=float, default=None,
                    help="with --mesh_clean: drop pieces of fewer faces than this fraction of the "
                         "largest piece's, in [0, 1] (default 0.01)")
    ap.add_argument("--mesh_max_hole", type=int, default=None,
                    help="with --mesh_clean: fill holes of at most this many boundary edges, 0 "
                         "(none, the default) or 3..128")
    ap.add_argument("--mesh_faces", type=int, default=None,
                    help="with --mesh: simplify the mesh to at most this many faces (>= 1) by "
                         "quadric edge-collapse decimation before it is written")
    ap.add_argument("--mesh_texture", action="store_true",
                    help="with --mesh: also texture the mesh from the reference views and write "
                         "<out>/mesh/<scan>.obj with its .mtl and atlas PNGs")
    ap.add_argument("--mesh_texture_level", action="store_true",
                    help="with --mesh_texture: level the colour seams between the atlas's charts "
                         "(global colour adjustment); only the page PNGs change")
    ap.add_argument("--mesh_refine", action="store_true",
                    help="with --mesh: move each vertex of the mesh along its normal to where the "
                         "reference views agree photometrically (after cleaning and simplifying, "
                         "before it is written, textured or scored)")
    ap.add_argument("--mesh_refine_iterations", type=int, default=None,
                    help="with --mesh_refine: refinement iterations, >= 1 (default 3)")
    ap.add_argument("--mesh_score", action="store_true",
                    help="with --mesh and --dtu_gt or --tnt_gt: also score the mesh as written "
                         "through its surface samples into <out>/mesh/<scan>_scores.json "
                         "(DTU) or <scan>_tnt.json")
    ap.add_argument("--remove_outliers", action="store_true",
                    help="remove statistical outliers from the fused cloud (and from Poisson's "
                         "points) on the GPU before it is written, scored or meshed: points whose "
                         "mean distance to their neighbours exceeds the cloud's mean by more than "
                         "--outlier_std standard deviations")
    ap.add_argument("--outlier_neighbours", type=int, default=None,
                    help="with --remove_outliers: neighbours per point, 1..64 (default 20)")
    ap.add_argument("--outlier_std", type=float, default=None,
                    help="with --remove_outliers: the standard-deviation ratio, > 0 (default 2.0)")
    a = ap.parse_args(argv)
    if getattr(a, "fusion", "reference") == "dynamic":
        ap.set_defaults(min_geo_consistent=None)                  # given explicitly?
        if ap.parse_args(argv).min_geo_consistent is not None:
            ap.error("--min_geo_consistent applies to --fusion reference only; the dynamic "
                     "rule sets its own view counts")
    if a.outlier_neighbours is not None and not a.remove_outliers:
        ap.error("--outlier_neighbours needs --remove_outliers")
    if a.outlier_std is not None and not a.remove_outliers:
        ap.error("--outlier_std needs --remove_outliers")
    if a.outlier_neighbours is not None and not 1 <= a.outlier_neighbours <= 64:
        ap.error("--outlier_neighbours must be in 1..64")
    if a.outlier_std is not None and not (math.isfinite(a.outlier_std) and a.outlier_std > 0):
        ap.error("--outlier_std must be a finite number > 0")
    if a.mesh_score and not a.mesh:
        ap.error("--mesh_score needs --mesh")
    if a.mesh_score and a.dtu_gt is None and a.tnt_gt is None:
        ap.error("--mesh_score needs a ground truth: --dtu_gt or --tnt_gt")
    if a.mesh_texture and not a.mesh:
        ap.error("--mesh_texture needs --mesh")
    if a.mesh_texture_level and not a.mesh_texture:
        ap.error("--mesh_texture_level needs --mesh_texture")
    if a.mesh_clean and not a.mesh:
        ap.error("--mesh_clean needs --mesh")
    if a.mesh_clean_ratio is not None and not a.mesh_clean:
        ap.error("--mesh_clean_ratio needs --mesh_clean")
    if a.mesh_max_hole is not None and not a.mesh_clean:
        ap.error("--mesh_max_hole needs --mesh_clean")
    if a.mesh_clean_ratio is not None and not (math.isfinite(a.mesh_clean_ratio)
                                               and 0 <= a.mesh_clean_ratio <= 1):
        ap.error("--mesh_clean_ratio must be in [0, 1]")
    if a.mesh_max_hole is not None and not (a.mesh_max_hole == 0 or 3 <= a.mesh_max_hole <= 128):
        ap.error("--mesh_max_hole must be 0 or in 3..128")
    if a.mesh_refine and not a.mesh:
        ap.error("--mesh_refine needs --mesh")
    if a.mesh_refine_iterations is not None and not a.mesh_refine:
        ap.error("--mesh_refine_iterations needs --mesh_refine")
    if a.mesh_refine_iterations is not None and a.mesh_refine_iterations < 1:
        ap.error("--mesh_refine_iterations must be >= 1")
    if a.mesh_faces is not None and not a.mesh:
        ap.error("--mesh_faces needs --mesh")
    if a.mesh_faces is not None and a.mesh_faces < 1:
        ap.error("--mesh_faces must be >= 1")
    if a.mesh_voxel is not None and not a.mesh_voxel > 0:
        ap.error("--mesh_voxel must be > 0")
    if a.mesh_method is not None and not a.mesh:
        ap.error("--mesh_method needs --mesh")
    if a.mesh_voxel is not None and a.mesh_method == "poisson":
        ap.error("--mesh_voxel applies to --mesh_method tsdf, not poisson")
    if a.poisson_depth is not None and a.mesh_method != "poisson":
        ap.error("--poisson_depth needs --mesh_method poisson")
    if a.poisson_depth is not None and not 6 <= a.poisson_depth <= 10:
        ap.error("--poisson_depth must be in 6..10")
    if a.poisson_point_weight is not None and a.mesh_method != "poisson":
        ap.error("--poisson_point_weight needs --mesh_method poisson")
    if a.poisson_point_weight is not None and not (math.isfinite(a.poisson_point_weight)
                                                   and a.poisson_point_weight >= 0):
        ap.error("--poisson_point_weight must be a finite number >= 0")
    a.mesh_method = a.mesh_method or "tsdf"
    if a.depth_interval is None:
        a.depth_interval = DEFAULT_DEPTH_INTERVAL[a.dataset_name]
    a.out_dir = a.out or os.path.join("results", a.dataset_name)
    return a


def _clean_options(a):
    """clean_mesh's options from --mesh_clean_ratio / --mesh_max_hole, or None without
    --mesh_clean."""
    if not a.mesh_clean:
        return None
    opts = dict(min_ratio=a.mesh_clean_ratio, max_hole=a.mesh_max_hole)
    return {k: v for k, v in opts.items() if v is not None}


def _refine_iterations(a):
    """refine_mesh's iterations from --mesh_refine_iterations (default refine.ITERATIONS), or
    None without --mesh_refine."""
    if not a.mesh_refine:
        return None
    from . import refine
    return refine.ITERATIONS if a.mesh_refine_iterations is None else a.mesh_refine_iterations


def _outlier_options(a):
    """filter options from --outlier_neighbours / --outlier_std, or None without
    --remove_outliers."""
    if not a.remove_outliers:
        return None
    opts = dict(k=a.outlier_neighbours, std_ratio=a.outlier_std)
    return {k: v for k, v in opts.items() if v is not None}


def main(argv=None):
    a = parse_args(argv)
    if a.dtu_gt is not None and a.dataset_name != "dtu":
        raise SystemExit("--dtu_gt applies to dtu only")
    if a.tnt_gt is not None and a.dataset_name != "colmap":
        raise SystemExit("--tnt_gt applies to colmap only")
    if a.image_dir is not None and a.dataset_name != "colmap":
        raise SystemExit("--image_dir applies to colmap only")
    if a.dataset_name == "dtu" and not a.scan:
        raise SystemExit("--scan is required for dtu")
    splits = {"tanks": TanksTestScan.SCANS, "blendedmvs": BlendedMVSTestScan.SPLITS}.get(a.dataset_name)
    if splits is not None and a.split not in splits:
        raise SystemExit(f"--split must be one of {sorted(splits)} for {a.dataset_name}")
    out_dir = a.out_dir
    from . import ABN
    from .models.mvsnet import CascadeMVSNet
    model = CascadeMVSNet(n_depths=a.n_depths, interval_ratios=a.interval_ratios,
                          num_groups=a.num_groups, norm_act=ABN, precision=a.precision,
                          depth_sampling=getattr(a, "depth_sampling", "uniform"))
    if a.ckpt:
        load_checkpoint(model, a.ckpt)
    model = model.eval().cuda()
    os.makedirs(os.path.join(out_dir, "points"), exist_ok=True)
    if a.mesh:
        os.makedirs(os.path.join(out_dir, "mesh"), exist_ok=True)
    for scan in open_scans(a):
        tnt = {}
        if a.tnt_gt is not None:
            tnt = dict(tnt_gt=a.tnt_gt, tnt_images=a.tnt_images, tnt_tau=a.tnt_tau,
                       tnt_seed=a.tnt_seed, run_dir=os.path.join(out_dir, scan.scan))
        out = run_scan(model, scan, a.depth_interval, a.conf, a.min_geo_consistent, a.skip,
                       a.max_ref_views, depth_dir=os.path.join(out_dir, "depth"),
                       ply_path=os.path.join(out_dir, "points", f"{scan.scan}.ply"), dtu_gt=a.dtu_gt,
                       dtu_seed=a.dtu_seed, save_visual=a.save_visual,
                       mesh_path=os.path.join(out_dir, "mesh", f"{scan.scan}.ply") if a.mesh else None,
                       mesh_voxel=a.mesh_voxel, mesh_method=a.mesh_method,
                       poisson_depth=a.poisson_depth,
                       poisson_point_weight=a.poisson_point_weight or 0.0,
                       mesh_faces=a.mesh_faces, mesh_texture=a.mesh_texture,
                       mesh_score=a.mesh_score, mesh_texture_level=a.mesh_texture_level,
                       mesh_clean=_clean_options(a),
                       fusion_rule=getattr(a, "fusion", "reference"),
                       outlier_filter=_outlier_options(a), mesh_refine=_refine_iterations(a), **tnt)
        print(f"{scan.scan} contains {len(out[0]) / 1e6:.2f} M points")
        if a.dtu_gt is not None:
            from .dtu_eval import _fmt
            print(_fmt(out[2]))
        if a.tnt_gt is not None:
            from .tnt_eval import _fmt
            print(_fmt(out[2]))
        if a.mesh_score:
            print(f"mesh {_fmt(out[3])}  ({out[3]['n_faces']} faces -> {out[3]['n_samples']} samples)")


if __name__ == "__main__":
    main()
