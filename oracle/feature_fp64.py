"""Float64 reference of FeatureNet's top-down kernels (csrc/fpn.cu: fpn_merge, fpn_level) and of
the x2 bilinear upsample they share with K4, with a per-element error bound, for per-element
checks.  The convolutions of FeatureNet (conv2d_rgb8, the planar 3x3 and the 5x5 stride-2
layers) are checked with oracle/conv3d_fp64.py.

Plain torch only (no casmvsnet_pl_b200 import, no F.interpolate / F.conv2d): source positions,
taps and sums are written out in float64 from the float32 inputs the kernels see.  The same
functions run on the CPU and on the GPU.  Tensors are channels-last: prev (N, h/2, w/2, C),
c (N, h, w, CLAT), outputs (N, h, w, C).

Bound per element, |y - y64| <= bound0 + eps * A, derived from the kernels' fp32 arithmetic
(u = 2^-24):

* Upsample position.  align_corners=True puts output row y at fy = y (hi - 1) / (h - 1) of the
  (hi = h/2)-row input.  The kernels round the scale (hi - 1) / (h - 1) and the product, so
  |fy' - fy| <= 2 u fy (1 + 2^-20) = dy; likewise dx.  Bilinear interpolation is Lipschitz in
  each coordinate with the largest difference of adjacent texels on its path; a position error
  below one texel keeps the path inside the 4x4 texels around the window, so the position term
  is L (dy + dx) with L that maximum per channel (as oracle/warp_cost_fp64._View does).  The
  clamped right and bottom taps extend the image by its last texel, which keeps it continuous.
* Blend.  ly = fy' - y0 is exact; each weight takes up to 3 roundings (1 - ly, 1 - lx, their
  product) and the weighted sum of 4 terms up to 7 in the unfused form: EPS_BLEND M with
  M = sum_i |w_i| |f_i|.
* Lateral and merge.  lat = lat_w c + lat_b, merge = up(prev) + lat: one fp32 fma chain seeded
  with the bias (fpn_merge: and the upsampled value), so the reduction term is eps A with
  A = sum |lat_w| |c| + |lat_b| + M.  A TF32-rounded store adds R_TF32 |y| / (1 - R_TF32).
* Level.  out = smooth3x3(merge) + smooth_b, zero padded.  The merge is not stored for level 0
  (the kernel keeps it in shared memory), so its bound is carried through the 3x3 sum:
  bound0 = sum |smooth_w| bound0_merge, and A = sum |smooth_w| (|merge| + A_merge) + |smooth_b|,
  so that one eps covers the merge's chain and the smoothing's.

Reports (``Report``) give the worst element by err / bound at (n, y, x, c) with x % 32, x % 16
(the fpn_level tile), x % 4 (conv2d_rgb8's four pixels per thread) and y % 16, the kernel and
float64 values, the smallest eps that would pass, and the loose share: the fraction of elements
whose bound exceeds LOOSE_REL of their magnitude A.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import warp_cost_fp64 as W
from oracle.conv3d_fp64 import CONV_PLANAR, R_TF32, TINY, conv3d_ref, pack_weight  # noqa: F401

ULP = 2.0 ** -24
SAFE = 1 + 2.0 ** -20               # second-order terms of the derived bounds
POS_REL = 2 * ULP * SAFE            # source position: rounded scale, rounded product
EPS_BLEND = 10 * ULP                # 3 roundings of the weights + 7 of the weighted sum
LOOSE_REL = W.LOOSE_REL


# ------------------------------------------------------------------------------- upsample
def up_positions(n_out, n_in, device="cpu"):
    """Exact float64 source positions i (n_in - 1) / (n_out - 1) of the align_corners x2
    upsample, and the bound on the kernels' fp32 positions."""
    i = torch.arange(n_out, dtype=torch.float64, device=device)
    f = i * (n_in - 1) / (n_out - 1) if n_in > 1 and n_out > 1 else torch.zeros_like(i)
    return f, POS_REL * f


def lipschitz_map(f):
    """f (N, hi, wi, C) float64 -> (N, hi, wi, C): at each window origin (y0, x0), the largest
    difference of adjacent texels over texels y0-1 .. y0+2, x0-1 .. x0+2."""
    e = torch.zeros_like(f)
    e[:, :, :-1] = (f[:, :, 1:] - f[:, :, :-1]).abs()
    e[:, :-1] = torch.maximum(e[:, :-1], (f[:, 1:] - f[:, :-1]).abs())
    ep = F.pad(e.permute(0, 3, 1, 2), (1, 2, 1, 2))
    return F.max_pool2d(ep, 4, stride=1).permute(0, 2, 3, 1)


def upsample2x(prev):
    """prev (N, hi, wi, C) -> float64 (N, 2hi, 2wi, C): the align_corners bilinear upsample,
    its bound without eps (position + blend) and the blend magnitude M = sum |w_i| |f_i|."""
    f = prev.double()
    N, hi, wi, C = f.shape
    h, w = 2 * hi, 2 * wi
    fy, dy = up_positions(h, hi, f.device)
    fx, dx = up_positions(w, wi, f.device)
    y0 = fy.floor().clamp(max=hi - 1).long()
    x0 = fx.floor().clamp(max=wi - 1).long()
    y1, x1 = (y0 + 1).clamp(max=hi - 1), (x0 + 1).clamp(max=wi - 1)
    ly = (fy - y0).view(1, h, 1, 1)
    lx = (fx - x0).view(1, 1, w, 1)
    r0, r1 = f[:, y0], f[:, y1]
    taps = (r0[:, :, x0], r0[:, :, x1], r1[:, :, x0], r1[:, :, x1])
    wts = ((1 - ly) * (1 - lx), (1 - ly) * lx, ly * (1 - lx), ly * lx)
    up = sum(wt * t for wt, t in zip(wts, taps))
    M = sum(wt * t.abs() for wt, t in zip(wts, taps))
    L = lipschitz_map(f)[:, y0][:, :, x0]
    bound0 = L * (dy.view(1, h, 1, 1) + dx.view(1, 1, w, 1)) + EPS_BLEND * M
    return up, bound0, M


# ------------------------------------------------------------------------------- merge, level
def lateral(c, lat_w, lat_b):
    """1x1 lateral + bias: c (N, h, w, CLAT), lat_w (32, CLAT) -> float64 (N, h, w, 32) and
    A = sum |lat_w| |c| + |lat_b|."""
    w64 = lat_w.detach().reshape(lat_w.shape[0], -1).to(device=c.device, dtype=torch.float64)
    b64 = lat_b.detach().to(device=c.device, dtype=torch.float64)
    c64 = c.double()
    return c64 @ w64.T + b64, c64.abs() @ w64.abs().T + b64.abs()


def merge_ref(prev, c, lat_w, lat_b):
    """up(prev) + lat_w c + lat_b (prev None: the lateral alone) -> y64, bound0, A."""
    lat, A = lateral(c, lat_w, lat_b)
    if prev is None:
        return lat, torch.zeros_like(lat), A
    up, b0, M = upsample2x(prev)
    return up + lat, b0, A + M


def level_ref(prev, c, lat_w, lat_b, sm_w, sm_b):
    """fpn_level: ((feat64, bound0, A) of the merge, (out64, bound0, A) of the smoothed
    output); sm_w (COUT, 32, 3, 3) torch layout."""
    feat, fb0, fA = merge_ref(prev, c, lat_w, lat_b)
    wp = pack_weight(sm_w, CONV_PLANAR).to(feat.device)
    wa = wp.abs()
    sb = sm_b.detach().to(device=feat.device, dtype=torch.float64)
    out = conv3d_ref(feat.unsqueeze(0), wp, CONV_PLANAR)[0] + sb
    b0 = conv3d_ref(fb0.unsqueeze(0), wa, CONV_PLANAR)[0]
    A = conv3d_ref((feat.abs() + fA).unsqueeze(0), wa, CONV_PLANAR)[0] + sb.abs()
    return (feat, fb0, fA), (out, b0, A)


# ------------------------------------------------------------------------------- reports
class Report(W.Report):
    """W.Report with the tile positions of FeatureNet's kernels in the description."""

    def describe(self):
        wv = self.worst
        at = dict(zip(self.names, wv["at"]))
        where = ", ".join(f"{k}={v}" for k, v in at.items())
        extra = ""
        if "x" in at:
            extra += f" x%32={at['x'] % 32} x%16={at['x'] % 16} x%4={at['x'] % 4}"
        if "y" in at:
            extra += f" y%16={at['y'] % 16}"
        if "d" in at:
            extra += f" plane={at['d']}"
        return (f"worst err/bound {self.ratio:.3e} at ({where}){extra}: got {wv['got']!r}, "
                f"float64 {wv['want']!r}, bound {wv['bound']:.3e}, A {wv['A']:.3e}; "
                f"eps needed {self.eps_needed:.3e} (eps {self.eps:.3e}); "
                f"loose share {self.loose_share:.2e}")


@torch.no_grad()
def check(y, y64, bound0, A, eps, tf32=False, names=("n", "y", "x", "c"), scale=None):
    """Kernel output y against float64 y64 with bound bound0 + eps A (+ the TF32 store)."""
    rep = Report(eps, tf32, names)
    rep.add(y, y64, bound0, A, (0,) * y64.dim(), A if scale is None else scale)
    return rep
