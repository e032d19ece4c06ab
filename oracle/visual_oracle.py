"""numpy restatement of csrc/visual.cu, the training panels (utils/visualization.py and the
image logging of train.py:107-114 in the original project), byte for byte.

Every step is float32 as in the original chain; the float32 -> uint8 cast is spelled out
(`np_u8`) rather than left to the platform: numpy on x86-64 truncates to int32 and keeps the low
byte, and a value outside [-2^31, 2^31) or NaN becomes INT_MIN, byte 0.
tests/golden/visual/cast.npz pins that rule against numpy's own cast.
"""
from __future__ import annotations

import numpy as np

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def colormaps():
    """{"JET", "BONE"} -> (256, 3) uint8 in cv2's BGR order, from the committed header."""
    import os
    import re
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                        "casmvsnet_pl_b200", "csrc", "colormap_table.h")
    src = open(path).read()
    out = {}
    for name, body in re.findall(r"kColormap(\w+)\[256\]\[3\] = \{(.*?)\n\};", src, flags=re.S):
        out[name.upper()] = np.array([int(v) for v in re.findall(r"\d+", body)], np.uint8).reshape(256, 3)
    return out


def np_u8(x):
    """numpy's float32 -> uint8 cast on x86-64."""
    t = np.asarray(x, np.float32).astype(np.float64)
    ok = (t >= -2.0 ** 31) & (t < 2.0 ** 31)
    i = np.trunc(np.where(ok, t, -2.0 ** 31)).astype(np.int64)
    return (i & 255).astype(np.uint8)


def unpreprocess(img):
    """(3,H,W) normalised float32 -> torchvision Normalize(mean=-m/s, std=1/s), float32."""
    mean = np.array([-m / s for m, s in zip(IMAGENET_MEAN, IMAGENET_STD)], np.float32)[:, None, None]
    std = np.array([1.0 / s for s in IMAGENET_STD], np.float32)[:, None, None]
    return (np.asarray(img, np.float32) - mean) / std


def image_panel(img):
    """-> (H,W,3) uint8: TensorBoard's u8((x * 255).clip(0, 255)) of the un-normalised image."""
    x = unpreprocess(img).transpose(1, 2, 0)
    return np_u8((x * np.float32(255)).clip(0, 255))


def depth_grey(depth):
    """visualize_depth's grey levels (H,W) uint8; no positive value -> all 0 (the original
    raises there)."""
    x = np.nan_to_num(np.asarray(depth, np.float32))
    pos = x[x > 0]
    if pos.size == 0:
        return np.zeros(x.shape, np.uint8)
    mi, ma = np.float32(pos.min()), np.float32(x.max())
    with np.errstate(over="ignore", invalid="ignore"):
        x = (x - mi) / (ma - mi + np.float32(1e-8))
        return np_u8(np.float32(255) * x)


def prob_grey(prob):
    return np_u8(np.float32(255) * np.asarray(prob, np.float32))


def colour(grey, name):
    """cv2.applyColorMap's BGR bytes read as RGB (the original's Image.fromarray)."""
    return colormaps()[name][grey]


def visualize_depth(depth):
    """(H,W) -> (H,W,3) uint8, the bytes of the original's visualize_depth (x 255)."""
    return colour(depth_grey(depth), "JET")


def visualize_prob(prob):
    return colour(prob_grey(prob), "BONE")


def masked(x, mask):
    """x * mask in float32, as torch multiplies a float tensor by a bool one (inf * 0 is NaN)."""
    with np.errstate(invalid="ignore"):
        return np.asarray(x, np.float32) * np.asarray(mask).astype(np.float32)


def training_panel(img, depth_gt, depth_pred, conf, mask):
    """-> (H, 4W, 3) uint8: image, depth_gt, depth_pred * mask, conf * mask side by side."""
    return np.concatenate([image_panel(img), visualize_depth(depth_gt),
                           visualize_depth(masked(depth_pred, mask)),
                           visualize_prob(masked(conf, mask))], axis=1)
