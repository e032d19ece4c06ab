"""Host restatement of torchvision's ColorJitter(brightness, contrast) on PIL RGB images, in
numpy, for the tests of casmvs_jitter_normalize_u8_fwd (never used by the package):

  pil_blend        Image.blend(im1, im2, alpha) per byte (libImaging/Blend.c): float32
                   t = in1 + alpha * (in2 - in1); truncated for 0 <= alpha <= 1, else clamped
                   to [0, 255] and truncated
  pil_luma         Image.convert("L"): (19595 R + 38470 G + 7471 B + 0x8000) >> 16
  contrast_mean    ImageEnhance.Contrast's grey level: int(histogram mean of L + 0.5), the mean
                   in double
  jitter_u8        ColorJitter's brightness (blend with black) and contrast (blend with the
                   grey level) in the drawn order
  normalize        ToTensor + Normalize of uint8 (H,W,3) -> float32 (3,H,W), torchvision's order
"""
from __future__ import annotations

import numpy as np

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def pil_blend(in1, in2, alpha):
    """uint8 arrays (broadcast) blended as Pillow does, alpha rounded to a C float."""
    a = np.float32(alpha)
    x1 = np.asarray(in1).astype(np.float32)
    d = (np.asarray(in2).astype(np.int32) - np.asarray(in1).astype(np.int32)).astype(np.float32)
    t = x1 + a * d                                   # two float32 roundings, no FMA
    if 0 <= a <= 1:
        return t.astype(np.uint8)
    return np.where(t <= 0, 0, np.where(t >= 255, 255, np.clip(t, 0, 255).astype(np.int32))).astype(np.uint8)


def pil_luma(img):
    """(...,3) uint8 -> (...) uint8, Pillow's RGB -> L."""
    x = np.asarray(img).astype(np.int64)
    return ((x[..., 0] * 19595 + x[..., 1] * 38470 + x[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def contrast_mean(img):
    l = pil_luma(img)
    return int(float(l.astype(np.int64).sum()) / l.size + 0.5)


def jitter_u8(img, brightness_first, b, c):
    """(H,W,3) uint8 after the brightness and contrast adjustments of ColorJitter."""
    img = np.asarray(img, dtype=np.uint8)
    if brightness_first:
        img = pil_blend(0, img, b)
        return pil_blend(contrast_mean(img), img, c)
    img = pil_blend(contrast_mean(img), img, c)
    return pil_blend(0, img, b)


def normalize(img_u8):
    """ToTensor + Normalize: x.float().div(255).sub(mean).div(std), per channel, float32."""
    x = np.asarray(img_u8, dtype=np.uint8).transpose(2, 0, 1).astype(np.float32)
    x = x / np.float32(255)
    mean = np.array(IMAGENET_MEAN, np.float32).reshape(3, 1, 1)
    std = np.array(IMAGENET_STD, np.float32).reshape(3, 1, 1)
    return ((x - mean) / std).astype(np.float32)


def jitter_normalize(imgs_u8, jitter):
    """(N,H,W,3) uint8 and (N,3) rows (brightness_first, b, c) -> (N,3,H,W) float32."""
    return np.stack([normalize(jitter_u8(im, bool(j[0]), float(j[1]), float(j[2])))
                     for im, j in zip(np.asarray(imgs_u8), np.asarray(jitter, np.float32))])
