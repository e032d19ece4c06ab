"""Record tests/golden/visual/*.npz from the REAL reference's panel code (needs the reference tree,
CASMVS_REFERENCE_ROOT or /root/reference; run from the repository root):

    python -m oracle.make_golden_visual

<case>.npz  inputs (img (3,H,W) normalised float32, depth_gt, depth_pred, conf (H,W) float32,
            mask (H,W) bool) and what the original's training_step makes of them:
            unpreprocessed = its T.Normalize(mean=-m/s, std=1/s)(img); vis_depth_gt =
            utils.visualize_depth(depth_gt); vis_depth_pred = visualize_depth(depth_pred * mask);
            vis_prob = visualize_prob(conf * mask); panel = the (H, 4W, 3) uint8 image that
            TensorBoard's summary.image stores for add_images of their stack, decoded from its
            PNG.  Where visualize_depth raises (no positive depth), `<name>_raises` is True and
            that output is the engine's rule instead: cv2's colour of grey level 0 everywhere,
            through the original's fromarray / ToTensor chain.
cast.npz    numpy's float32 -> uint8 cast of values across the negative range, past 2^31 and at
            the int32 limits, inf and NaN (the cast the panels' grey levels go through).
"""
from __future__ import annotations

import io as _io
import os

import numpy as np
import torch

from oracle.ref_loader import REFERENCE_ROOT, reference_available

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "visual")
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _smooth(rng, H, W, k=6, block=4):
    """A smooth field in [0, 1], a few random cosines, constant over block x block tiles (keeps
    the recorded maps small when compressed)."""
    y, x = (np.mgrid[0:H, 0:W] // block * block).astype(np.float64)
    f = np.zeros((H, W))
    for _ in range(k):
        a, b = rng.uniform(0.5, 4, 2) * np.pi / np.array([W, H]), rng.uniform(0, 2 * np.pi)
        f += np.cos(a[0] * x + a[1] * y + b)
    return (f - f.min()) / (f.max() - f.min())


def _image(rng, H, W):
    """A uint8 RGB image normalised as the data readers do: (u8 / 255 - m) / s in float32."""
    u8 = np.stack([np.round(255 * _smooth(rng, H, W)) for _ in range(3)]).astype(np.uint8)
    m = np.array(MEAN, np.float32)[:, None, None]
    s = np.array(STD, np.float32)[:, None, None]
    return ((u8.astype(np.float32) / np.float32(255)) - m) / s


def _holes(rng, H, W, n):
    keep = np.ones((H, W), bool)
    for _ in range(n):
        cy, cx = rng.integers(0, H), rng.integers(0, W)
        r = rng.integers(H // 20 + 1, H // 6 + 2)
        y, x = np.ogrid[0:H, 0:W]
        keep &= (y - cy) ** 2 + (x - cx) ** 2 > r * r
    return keep


def _q(x, step):
    """Quantise to multiples of `step` (keeps the recorded maps small when compressed)."""
    return (np.round(np.asarray(x, np.float64) / step) * step).astype(np.float32)


def case_scene(seed, H, W, dmin, dmax, step):
    rng = np.random.default_rng(seed)
    keep = _holes(rng, H, W, 8)
    gt = _q(dmin + (dmax - dmin) * _smooth(rng, H, W), step) * keep
    pred = _q(gt + (dmax - dmin) * 0.02 * (_smooth(rng, H, W) - 0.5), step)
    pred[~keep] = _q(dmin + (dmax - dmin) * _smooth(rng, H, W), step)[~keep]
    conf = _q(_smooth(rng, H, W), 1.0 / 1024)
    return dict(img=_image(rng, H, W), depth_gt=gt.astype(np.float32), depth_pred=pred,
                conf=conf, mask=gt > dmin * 0.5)


def _small(seed, H=48, W=64):
    rng = np.random.default_rng(seed)
    s = case_scene(seed, H, W, 425.0, 935.0, 1.0 / 16)
    return rng, s


def case_nan_inf():
    rng, s = _small(1)
    for key in ("depth_gt", "depth_pred", "conf"):
        flat = s[key].reshape(-1)
        idx = rng.choice(flat.size, 60, replace=False)
        flat[idx[:20]] = np.nan
        flat[idx[20:40]] = np.inf
        flat[idx[40:]] = -np.inf
    return s


def case_nan_pred():
    """NaN and +-inf only in the prediction: the gt panel keeps its usual range."""
    rng, s = _small(2)
    flat = s["depth_pred"].reshape(-1)
    idx = rng.choice(flat.size, 90, replace=False)
    flat[idx[:30]], flat[idx[30:60]], flat[idx[60:]] = np.nan, np.inf, -np.inf
    return s


def case_constant():
    _, s = _small(3)
    s["depth_gt"] = np.where(s["mask"], np.float32(500.0), np.float32(0.0)).astype(np.float32)
    s["depth_pred"] = np.full_like(s["depth_gt"], 712.25)
    return s


def case_conf_levels():
    _, s = _small(4)
    H, W = s["conf"].shape
    one = np.float32(1.0)
    special = [np.nextafter(one, np.float32(2)), one + np.float32(1e-6), np.float32(1.003),
               np.float32(1.004), np.float32(1.0039216), np.float32(2.0), np.float32(-1e-6),
               np.float32(-0.5), np.nextafter(np.float32(0), np.float32(1)), np.float32(0.5)]
    levels = np.arange(256, dtype=np.float32) / np.float32(255)
    vals = np.concatenate([levels, np.nextafter(levels, np.float32(2)),
                           np.nextafter(levels, np.float32(-1)), np.array(special, np.float32)])
    s["conf"] = np.resize(vals, H * W).reshape(H, W).astype(np.float32)
    s["mask"][:, :3] = False
    return s


def case_image_range():
    rng, s = _small(5)
    s["img"] = _q(rng.uniform(-4.0, 4.0, s["img"].shape), 1.0 / 512)
    return s


def case_wide_negative():
    """Grey levels of masked-out and negative depths far below the range: the cast wraps."""
    rng, s = _small(6)
    H, W = s["depth_gt"].shape
    mags = np.float32(10.0) ** rng.uniform(-1, 13, H * W).astype(np.float32)
    s["depth_gt"] = (-mags).reshape(H, W).astype(np.float32)
    s["depth_gt"][0, :4] = [1.0, 256.0, -np.finfo(np.float32).max, -2.0 ** 31]
    s["depth_pred"] = _q(rng.uniform(1.0, 3.0, (H, W)), 1.0 / 8)
    return s


def case_no_positive():
    _, s = _small(7)
    s["depth_gt"] = -np.abs(s["depth_gt"])
    s["mask"][:] = False
    return s


def cases():
    return {
        "dtu_640x512": case_scene(10, 512, 640, 425.0, 935.0, 1.0 / 16),
        "blendedmvs_768x576": case_scene(11, 576, 768, 2.5, 61.0, 1.0 / 256),
        "nan_inf": case_nan_inf(),
        "nan_pred": case_nan_pred(),
        "constant": case_constant(),
        "conf_levels": case_conf_levels(),
        "image_range": case_image_range(),
        "wide_negative": case_wide_negative(),
        "no_positive": case_no_positive(),
    }


def cast_table():
    rng = np.random.default_rng(0)
    neg = -(np.float32(2.0) ** rng.uniform(-2, 40, 4000).astype(np.float32))
    edges = []
    for e in (2.0 ** 31, 2.0 ** 32, 2.0 ** 63, 256.0, 128.0, 1.0):
        for v in (np.float32(e), np.float32(-e)):
            edges += [np.nextafter(v, np.float32(0)), v, np.nextafter(v, -v * 2)]
    x = np.concatenate([neg, -neg, np.array(edges, np.float32),
                        np.array([np.inf, -np.inf, np.nan, -0.0, 3.4e38, -3.4e38, -212.7, -1e6],
                                 np.float32)]).astype(np.float32)
    with np.errstate(invalid="ignore"):
        return {"x": x, "u8": x.astype(np.uint8)}


def record(s):
    import cv2
    import torchvision.transforms as T
    from PIL import Image
    from torch.utils.tensorboard.summary import image as tb_image

    from oracle.make_golden_train import reference_utils
    u = reference_utils()
    unpre = T.Normalize(mean=[-0.485 / 0.229, -0.456 / 0.224, -0.406 / 0.225],
                        std=[1 / 0.229, 1 / 0.224, 1 / 0.225])      # train.py:33-34
    mask = torch.from_numpy(s["mask"])
    out = dict(s)
    img_ = unpre(torch.from_numpy(s["img"].copy()))
    panels = [img_]
    for name, fn, x in (("vis_depth_gt", u.visualize_depth, torch.from_numpy(s["depth_gt"])),
                        ("vis_depth_pred", u.visualize_depth, torch.from_numpy(s["depth_pred"]) * mask),
                        ("vis_prob", u.visualize_prob, torch.from_numpy(s["conf"]) * mask)):
        try:
            with np.errstate(invalid="ignore", over="ignore"):
                v = fn(x)
            out[name + "_raises"] = np.bool_(False)
        except ValueError:
            grey0 = cv2.applyColorMap(np.zeros(s["mask"].shape, np.uint8), cv2.COLORMAP_JET)
            v = T.ToTensor()(Image.fromarray(grey0))
            out[name + "_raises"] = np.bool_(True)
        out[name] = v.numpy()
        panels.append(v)
    stack = torch.stack(panels)
    summ = tb_image("train/image_GT_pred_prob", stack, dataformats="NCHW")
    png = summ.value[0].image.encoded_image_string
    out["panel"] = np.asarray(Image.open(_io.BytesIO(png)).convert("RGB"))
    out["unpreprocessed"] = img_.numpy()
    return out


def main():
    if not reference_available():
        raise SystemExit(f"reference tree not found at {REFERENCE_ROOT}")
    os.makedirs(OUT, exist_ok=True)
    for name, s in cases().items():
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **record(s))
    np.savez_compressed(os.path.join(OUT, "cast.npz"), **cast_table())
    print("wrote", sorted(os.listdir(OUT)))


if __name__ == "__main__":
    import warnings
    warnings.filterwarnings("ignore")
    main()
