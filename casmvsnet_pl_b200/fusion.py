"""GPU geometric-consistency filter, depth / colour refinement and point-cloud fusion
(SURVEY.md 8 f-3) — the step right after the hot path, consumer of depth_0 / confidence_2.

Replaces the CPU code of the reference's eval.py:
    xy_ref2src / xy_src2ref / check_geo_consistency      eval.py:113-182   (numba + cv2.remap)
    per-view masking, averaging, back-projection         eval.py:262-318
    the scan loop with its refined-view cache            eval.py:245-330
    PLY output                                           eval.py:337-350   (plyfile)
One kernel launch per reference view (csrc/fusion.cu) walks all its source views; depth maps,
confidence maps and images of a scan stay resident in HBM, so nothing goes through PFM files.
Arithmetic is fp32 like the reference's (float32 numpy + numba); images are float32 (the
reference remaps uint8 images, i.e. rounds the warped colours to integers first — colours here
can differ by < 1 grey level, geometry is unaffected).

Two consistency rules (``rule=``): "reference", eval.py's fixed check (a source agrees within
1 px and 1 % relative depth; keep a pixel that at least min_geo_consistent sources agree on), and
"dynamic", the count-based dynamic consistency check of D2HC-RMVSNet (Yan et al., ECCV 2020):
keep a pixel when, for some level k in DYNAMIC_LEVELS, at least k sources agree within k / 4 px
and k / 1300 relative depth (tight agreement from few views, or loose agreement from many).
csrc/fusion.cu states the rule in full.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib

RULES = ("reference", "dynamic")
# The dynamic rule's constants, as csrc/fusion.cu states them (kDynLevelMin, kDynLevelMax,
# kDynPixDiv, kDynDepDiv): level k is e_pix < (k / DYNAMIC_PIX_DIV)^2 and
# e_dep < float32(k / DYNAMIC_DEP_DIV), for k in DYNAMIC_LEVELS.
DYNAMIC_LEVELS = range(2, 11)
DYNAMIC_PIX_DIV = 4
DYNAMIC_DEP_DIV = 1300


def _check_rule(rule):
    if rule not in RULES:
        raise ValueError(f"rule must be one of {RULES}, got {rule!r}")


def _rel(P_a, P_b):
    """(P_a @ inv(P_b))[:3] in float32 numpy, like eval.py:120,136."""
    P_a = np.asarray(P_a, dtype=np.float32)
    P_b = np.asarray(P_b, dtype=np.float32)
    return np.ascontiguousarray((P_a @ np.ascontiguousarray(np.linalg.inv(P_b)))[:3], dtype=np.float32)


def refine_ref_view(depth_ref, P_world2ref, depth_srcs, P_world2srcs, image_ref=None,
                    image_srcs=None, proba_ref=None, conf=0.999, min_geo_consistent=5,
                    want_points=True, debug=False, rule="reference"):
    """One reference view of eval.py:262-318.

    depth_ref (H,W), depth_srcs [S x (H,W)], image_ref (H,W,3) / image_srcs [S x (H,W,3)]
    float32 CUDA tensors (images optional), proba_ref (H/4,W/4) = confidence_2 (optional: no
    confidence mask), P_* (4,4) float32 world->pixel matrices (numpy / CPU tensors).
    Returns dict: depth_refined (H,W), image_refined (H,W,3)|None, geo_count (H,W) int32,
    mask_final (H,W) bool, points (H,W,3)|None [+ reproj (S,H,W), mask (S,H,W) with debug].
    rule="dynamic" applies the dynamic consistency check (casmvs_geo_fuse_dynamic_fwd) in place
    of eval.py's: min_geo_consistent is then ignored, geo_count counts the sources consistent at
    the loosest level, and debug returns level (S,H,W) uint8, each source's least consistent
    level (0: none), in place of mask."""
    _check_rule(rule)
    if not depth_ref.is_cuda:
        raise _lib.CasMVSError("fusion runs on the GPU (no CPU fallback)")
    dev = depth_ref.device
    H, W = depth_ref.shape
    S = len(depth_srcs)
    f32 = dict(device=dev, dtype=torch.float32)
    depth_ref = depth_ref.contiguous()
    srcs = [d.contiguous() for d in depth_srcs]
    imgs = [i.contiguous() for i in image_srcs] if (image_srcs is not None and image_ref is not None) else None
    P_ref = np.asarray(P_world2ref, dtype=np.float32)
    rs = np.stack([_rel(P, P_ref) for P in P_world2srcs]).reshape(-1) if S else np.zeros(0, np.float32)
    sr = np.stack([_rel(P_ref, P) for P in P_world2srcs]).reshape(-1) if S else np.zeros(0, np.float32)
    ref2world = torch.from_numpy(np.ascontiguousarray(np.linalg.inv(P_ref), dtype=np.float32)).to(dev)
    out = dict(depth_refined=torch.empty(H, W, **f32),
               image_refined=torch.empty(H, W, 3, **f32) if image_ref is not None else None,
               geo_count=torch.empty(H, W, device=dev, dtype=torch.int32),
               mask_final=torch.empty(H, W, device=dev, dtype=torch.uint8),
               points=torch.empty(H, W, 3, **f32) if want_points else None)
    if debug:
        out["reproj"] = torch.empty(S, H, W, **f32)
        out["mask" if rule == "reference" else "level"] = torch.empty(S, H, W, device=dev,
                                                                      dtype=torch.uint8)

    def p(t):
        return ctypes.c_void_p(t.data_ptr()) if t is not None else None
    ptr_arr = ctypes.c_void_p * max(S, 1)
    d_arr = ptr_arr(*[d.data_ptr() for d in srcs]) if S else ptr_arr()
    i_arr = ptr_arr(*[i.data_ptr() for i in imgs]) if imgs else None
    with torch.cuda.device(dev):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        inputs = (p(depth_ref), p(image_ref.contiguous() if image_ref is not None else None),
                  p(proba_ref.contiguous() if proba_ref is not None else None), d_arr, i_arr,
                  rs.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                  sr.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), p(ref2world), S, H, W,
                  float(conf))
        outputs = (p(out["depth_refined"]), p(out["image_refined"]), p(out["geo_count"]),
                   p(out["mask_final"]), p(out["points"]), p(out.get("reproj")))
        if rule == "reference":
            _lib.check(_lib.load().casmvs_geo_fuse_fwd(
                *inputs, int(min_geo_consistent), *outputs, p(out.get("mask")), st), "geo_fuse")
        else:
            _lib.check(_lib.load().casmvs_geo_fuse_dynamic_fwd(
                *inputs, *outputs, p(out.get("level")), st), "geo_fuse_dynamic")
    out["mask_final"] = out["mask_final"].bool()
    if debug and rule == "reference":
        out["mask"] = out["mask"].bool()
    return out


def fuse_scan(metas, depths, probas, images, proj_mats, conf=0.999, min_geo_consistent=5, skip=1,
              max_ref_views=400, collect=None, rule="reference"):
    """The scan loop of eval.py:245-330.  metas: [(ref_vid, [src_vids])] in pair-file order;
    depths[vid] (H,W), probas[vid] (H/4,W/4), images[vid] (H,W,3) float32 RGB CUDA tensors;
    proj_mats[vid] (4,4) finest-level world->pixel.  Like the reference, a view that has been a
    reference view is used in its REFINED form (depth averaged over consistent views, colours
    rounded to uint8 as its PNG round trip does) by later reference views, and a source view's
    raw depth is cached on first use.  Returns (xyz (N,3) float32, rgb (N,3) uint8) on the GPU.
    With `collect` (a list), one dict per fused reference view is appended to it, in order, for
    meshing: depth (H,W) = refined depth where mask_final else 0, image = image_refined (H,W,3),
    P (4,4) and points = the world points of every masked pixel (not thinned by `skip`).
    `rule` is refine_ref_view's: with "dynamic", min_geo_consistent is ignored; the scan loop,
    the cache and the outputs are the same for both rules."""
    _check_rule(rule)
    image_refined, depth_refined = {}, {}
    vs, cs = [], []
    for ref_vid, src_vids in metas[:max_ref_views]:
        if ref_vid not in depths:
            continue                                   # eval.py:319-322: no prediction for it
        if ref_vid in image_refined:
            image_ref, depth_ref = image_refined[ref_vid], depth_refined[ref_vid]
        else:
            image_ref, depth_ref = images[ref_vid], depths[ref_vid]
        d_srcs, i_srcs, P_srcs = [], [], []
        missing = False
        for sv in src_vids:
            if sv in image_refined:
                i_srcs.append(image_refined[sv]); d_srcs.append(depth_refined[sv])
            elif sv in depths:
                depth_refined[sv] = depths[sv]
                i_srcs.append(images[sv]); d_srcs.append(depths[sv])
            else:
                missing = True                         # FileNotFoundError path of eval.py:319
                break
            P_srcs.append(proj_mats[sv])
        if missing:
            continue
        r = refine_ref_view(depth_ref, proj_mats[ref_vid], d_srcs, P_srcs, image_ref, i_srcs,
                            probas[ref_vid], conf, min_geo_consistent, rule=rule)
        depth_refined[ref_vid] = r["depth_refined"]
        # cv2.imwrite + cv2.imread of the refined image (eval.py:305-306): uint8, round half even
        image_refined[ref_vid] = torch.round(r["image_refined"]).clamp_(0, 255)
        m = r["mask_final"]
        vs.append(r["points"][m][::skip])
        cs.append(r["image_refined"][m][::skip])
        if collect is not None:
            collect.append(dict(depth=torch.where(m, r["depth_refined"], 0.0),
                                image=r["image_refined"], P=np.asarray(proj_mats[ref_vid], np.float32),
                                points=vs[-1] if skip == 1 else r["points"][m]))
    if not vs:
        dev = next(iter(depths.values())).device
        return torch.zeros(0, 3, device=dev), torch.zeros(0, 3, device=dev, dtype=torch.uint8)
    return torch.cat(vs).float(), torch.cat(cs).to(torch.uint8)      # .astype(np.uint8) truncates


def write_ply(path, xyz, rgb):
    """Binary little-endian PLY with the vertex layout eval.py:337-350 writes through plyfile:
    float x, y, z + uchar red, green, blue."""
    xyz = np.ascontiguousarray(xyz.detach().cpu().numpy() if torch.is_tensor(xyz) else xyz, np.float32)
    rgb = np.ascontiguousarray(rgb.detach().cpu().numpy() if torch.is_tensor(rgb) else rgb, np.uint8)
    n = len(xyz)
    v = np.empty(n, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"),
                           ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    v["x"], v["y"], v["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    v["red"], v["green"], v["blue"] = rgb[:, 0], rgb[:, 1], rgb[:, 2]
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {n}\nproperty float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        v.tofile(f)
