"""CPU oracle of the device resamplers (csrc/resize.cu): numpy restatements, in int64, of

  pil_bilinear(img, wh)   Pillow Image.resize(wh, Image.BILINEAR) on 8-bit RGB (Resample.c:
                          precompute_coeffs, normalize_coeffs_8bpc, ImagingResampleHorizontal_8bpc /
                          ImagingResampleVertical_8bpc; a pass is skipped when its size is unchanged)
  cv2_linear(img, wh)     cv2.resize(img, wh, interpolation=cv2.INTER_LINEAR) on 8-bit images
                          (resize.cpp: 11-bit weights, HResizeLinear, and the uchar specialisation of
                          VResizeLinear, whose vector and scalar forms compute
                          (((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2)

written from the libraries' documented arithmetic, independently of casmvsnet_pl_b200/io.py's
table builders.  tests/test_scan_ingest.py pins both against the installed Pillow / cv2.
"""
import math

import numpy as np

PRECISION_BITS = 22


def _pil_coeffs(insz, outsz):
    scale = insz / outsz
    fs = max(scale, 1.0)
    support, ss = fs, 1.0 / fs
    out = []
    for xx in range(outsz):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), insz) - xmin
        w = [max(0.0, 1.0 - abs((x + xmin - center + 0.5) * ss)) for x in range(xmax)]
        ww = 0.0
        for v in w:                       # sequential double sum, like the C loop
            ww += v
        w = [v / ww if ww != 0 else v for v in w]
        k = [int(math.floor(0.5 + v * (1 << PRECISION_BITS))) if v >= 0
             else int(math.ceil(-0.5 + v * (1 << PRECISION_BITS))) for v in w]
        out.append((xmin, k))
    return out


def _pil_pass(a, outsz, axis):
    a = np.moveaxis(a, axis, 0).astype(np.int64)
    res = np.empty((outsz,) + a.shape[1:], np.int64)
    for i, (xmin, k) in enumerate(_pil_coeffs(a.shape[0], outsz)):
        s = np.full(a.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
        for x, kx in enumerate(k):
            s += a[xmin + x] * kx
        res[i] = np.clip(s >> PRECISION_BITS, 0, 255)
    return np.moveaxis(res, 0, axis).astype(np.uint8)


def pil_bilinear(img, wh):
    """(H,W,C) uint8 -> (h,w,C) uint8 (horizontal pass first, then vertical)."""
    w, h = wh
    t = np.asarray(img, np.uint8)
    if w != t.shape[1]:
        t = _pil_pass(t, w, 1)
    if h != t.shape[0]:
        t = _pil_pass(t, h, 0)
    return t.copy()


def _cv_taps(insz, outsz, clamp):
    scale = 1.0 / (outsz / insz)
    f = ((np.arange(outsz, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp:                              # only the x taps are clamped (xmin / xmax)
        lo = s < 0
        f[lo], s[lo] = 0, 0
        hi = s >= insz - 1
        f[hi], s[hi] = 0, insz - 1
    a1 = np.rint(f * np.float32(2048)).astype(np.int64)
    a0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    return np.clip(s, 0, insz - 1), np.clip(s + 1, 0, insz - 1), a0, a1


def cv2_linear(img, wh):
    """(H,W,C) uint8 -> (h,w,C) uint8."""
    w, h = wh
    img = np.asarray(img, np.uint8)
    H, W = img.shape[:2]
    if (w, h) == (W, H):
        return img.copy()
    x0, x1, a0, a1 = _cv_taps(W, w, True)
    y0, y1, b0, b1 = _cv_taps(H, h, False)
    I = img.astype(np.int64)
    rows = I[:, x0] * a0[None, :, None] + I[:, x1] * a1[None, :, None]
    v = (((rows[y0] >> 4) * b0[:, None, None]) >> 16) + (((rows[y1] >> 4) * b1[:, None, None]) >> 16)
    return ((v + 2) >> 2).astype(np.uint8)
