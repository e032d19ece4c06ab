"""Float64 restatement of the self-supervised photometric loss (csrc/photo_loss.cu,
casmvs_photo_loss_fwd / _bwd) and its gradient, for per-element checks.

Plain torch only (no casmvsnet_pl_b200 import), on whatever device the inputs are.  Bilinear
sampling uses explicit taps (x0 = floor(u), tap x0 + 1 clamped to w - 1), not grid_sample, and
the gradient is torch autograd of this float64 expression.  `photo_loss` takes an optional
selection per level, so that the loss and gradient can be evaluated for the kernel's own
selection wherever near-ties make more than one selection admissible (the margin and bound of
`LevelResult` say where the float64 selection is unambiguous).

Bounds.  The kernel evaluates the warp in float32: each coordinate of p = R (x, y, 1) + T / d
carries at most ~4 ulp of the sum of its terms' magnitudes, so u = p_x / p_z is within
du = 4 eps (|p_x|_terms + |u| |p_z|_terms) / p_z + eps |u|, likewise v.  Un-normalised images
lie in [0, 1], so a bilinear sample moves by at most du + dv, plus ~4 ulp of rounding.  e's
bound is then sum over the window's samples of |de/dy| times that, plus a floor of 64 eps for
the float32 evaluation of SSIM (centred sums of 9 values in [0, 1]).
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
ALPHA = 0.85
C1 = 0.01 ** 2
C2 = 0.03 ** 2
EPS32 = 2.0 ** -24
E_FLOOR = 64 * EPS32


def level_images(imgs, l):
    """imgs (B,V,3,H,W) normalised -> float64 un-normalised level-l images (strided subsample)."""
    x = imgs.double()[..., :: 1 << l, :: 1 << l]
    mean = torch.tensor(MEAN, dtype=torch.float64, device=x.device).view(3, 1, 1)
    std = torch.tensor(STD, dtype=torch.float64, device=x.device).view(3, 1, 1)
    return x * std + mean


def warp(depth, P, w, h):
    """depth (B,h,w), P (B,S,3,4) -> u, v, valid, du, dv (B,S,h,w), float64, differentiable in depth."""
    B = depth.shape[0]
    dev = depth.device
    ys, xs = torch.meshgrid(torch.arange(h, device=dev, dtype=torch.float64),
                            torch.arange(w, device=dev, dtype=torch.float64), indexing="ij")
    d = depth.double()[:, None]
    ok_d = torch.isfinite(d) & (d > 0)
    inv = 1.0 / torch.where(ok_d, d, torch.ones_like(d))
    P = P.double()

    def row(r):
        m = P[:, :, r, :, None, None]
        terms = m[:, :, 0] * xs, m[:, :, 1] * ys, m[:, :, 2].expand(B, -1, h, w), m[:, :, 3] * inv
        return sum(terms), sum(t.abs() for t in terms)
    px, ax = row(0)
    py, ay = row(1)
    pz, az = row(2)
    ok_z = pz > 1e-7
    pzs = torch.where(ok_z, pz, torch.ones_like(pz))
    u, v = px / pzs, py / pzs
    valid = ok_d & ok_z & (u >= 0) & (u <= w - 1) & (v >= 0) & (v <= h - 1)
    du = (4 * EPS32 * (ax + u.abs() * az) / pzs + EPS32 * u.abs()).detach()
    dv = (4 * EPS32 * (ay + v.abs() * az) / pzs + EPS32 * v.abs()).detach()
    return u, v, valid, du, dv


def sample(img, u, v, valid):
    """img (B,S,3,h,w), u / v (B,S,h,w) -> (B,S,3,h,w) bilinear with explicit taps (0 invalid)."""
    B, S, C, h, w = img.shape
    uu = torch.where(valid, u, torch.zeros_like(u))
    vv = torch.where(valid, v, torch.zeros_like(v))
    x0 = torch.floor(uu).detach()
    y0 = torch.floor(vv).detach()
    fx, fy = uu - x0, vv - y0
    x0, y0 = x0.long(), y0.long()
    x1, y1 = (x0 + 1).clamp(max=w - 1), (y0 + 1).clamp(max=h - 1)
    flat = img.reshape(B, S, C, h * w)

    def tap(yy, xx):
        idx = (yy * w + xx).reshape(B, S, 1, h * w).expand(B, S, C, h * w)
        return flat.gather(3, idx).reshape(B, S, C, h, w)
    fx, fy = fx[:, :, None], fy[:, :, None]
    top = tap(y0, x0) * (1 - fx) + tap(y0, x1) * fx
    bot = tap(y1, x0) * (1 - fx) + tap(y1, x1) * fx
    out = top * (1 - fy) + bot * fy
    return torch.where(valid[:, :, None], out, torch.zeros_like(out))


def _win(t):
    """(..., h, w) -> (9, ..., h-2, w-2): the 3x3 window of every interior pixel."""
    h, w = t.shape[-2:]
    return torch.stack([t[..., j:h - 2 + j, i:w - 2 + i] for j in range(3) for i in range(3)])


@dataclass
class LevelResult:
    e: torch.Tensor          # (B,S,h,w) float64, NaN where not valid
    valid: torch.Tensor      # (B,S,h,w) bool
    e_bound: torch.Tensor    # (B,S,h,w) bound on |e_kernel - e| where valid
    selected: torch.Tensor   # (B,S,h,w) bool, the float64 selection (or the given one)
    margin: torch.Tensor     # (B,h,w) gap between the K-th and (K+1)-th valid e (inf if none)
    kink: torch.Tensor       # (B,h,w) the gradient at p may jump within float32's rounding
    loss_q: torch.Tensor     # (B,h,w), NaN where no source is valid
    P: torch.Tensor
    S: torch.Tensor
    N: torch.Tensor


def level_loss(depth, imgs, P, dint, ratio, l, topk, selected=None):
    """One level.  depth (B,h,w) (may require grad), imgs (B,V,3,H,W), P (B,S,3,4) of level l,
    dint (B,).  `selected` (B,S,h,w) bool replaces the float64 top-K selection."""
    I = level_images(imgs, l)
    B, V, _, h, w = I.shape
    S = V - 1
    ref, src = I[:, 0], I[:, 1:]
    u, v, ok, du, dv = warp(depth, P, w, h)
    y = sample(src, u, v, ok)                                    # (B,S,3,h,w)
    x = ref[:, None].expand_as(y)
    okw = _win(ok).all(0)                                        # (B,S,h-2,w-2)
    X, Y = _win(x), _win(y)                                      # (9,B,S,3,h-2,w-2)
    mx, my = X.mean(0), Y.mean(0)
    sxx = ((X - mx) ** 2).mean(0)
    syy = ((Y - my) ** 2).mean(0)
    sxy = ((X - mx) * (Y - my)).mean(0)
    a1, a2 = 2 * mx * my + C1, 2 * sxy + C2
    b1, b2 = mx ** 2 + my ** 2 + C1, sxx + syy + C2
    ssim = a1 * a2 / (b1 * b2)
    xc, yc = X[4], Y[4]
    e_in = ALPHA * ((1 - ssim) / 2).mean(2) + (1 - ALPHA) * (xc - yc).abs().mean(2)
    okw = okw & torch.isfinite(e_in)           # a non-finite e cannot be ordered: not valid
    with torch.no_grad():      # |de/dy_i| of every window sample, times the sample's bound
        k = (2.0 / 9.0) * ALPHA / 6.0
        ib = 1.0 / (b1 * b2)
        ca = mx * a2 * ib - my * ssim / b1 - mx * a1 * ib + my * ssim / b2
        cb, cc = a1 * ib, -ssim / b2
        dy = _win((du + dv)[:, :, None].expand_as(y)) + 4 * EPS32
        sens = (k * (ca + cb * X + cc * Y)).abs()
        sens[4] += (1 - ALPHA) / 3
        bound = (sens * dy).sum(0).sum(2) + E_FLOOR
    nan = torch.full((), float("nan"), dtype=torch.float64, device=depth.device)
    e = torch.full((B, S, h, w), float("nan"), dtype=torch.float64, device=depth.device)
    valid = torch.zeros(B, S, h, w, dtype=torch.bool, device=depth.device)
    e_bound = torch.zeros(B, S, h, w, dtype=torch.float64, device=depth.device)
    e[..., 1:-1, 1:-1] = torch.where(okw, e_in, nan)
    valid[..., 1:-1, 1:-1] = okw
    e_bound[..., 1:-1, 1:-1] = bound
    n_valid = valid.sum(1)
    with torch.no_grad():
        key = torch.where(valid, e.detach(), torch.full_like(e.detach(), float("inf")))
        order = torch.argsort(key, dim=1, stable=True)
        rank = torch.argsort(order, dim=1)
        srt = key.gather(1, order)
        kk = torch.clamp(n_valid, max=topk)
        own = rank < kk[:, None]
        if S > topk:
            gap = srt[:, topk] - srt[:, topk - 1]
            margin = torch.where(n_valid > topk, gap, torch.full_like(gap, float("inf")))
        else:
            margin = torch.full_like(srt[:, 0], float("inf"))
    sel = own if selected is None else selected.to(depth.device).bool()
    nsel = sel.sum(1)
    e0 = torch.where(sel, e, torch.zeros_like(e))
    loss_q = torch.where(nsel > 0, e0.sum(1) / nsel.clamp(min=1), nan)
    has = n_valid > 0
    N = has.sum().double()
    Pl = torch.where(has, torch.nan_to_num(loss_q, nan=0.0), torch.zeros_like(loss_q)).sum()
    Pl = Pl / N if N > 0 else Pl * 0
    # smoothness
    dhat = depth.double() / (dint.double().view(-1, 1, 1) * ratio)
    with torch.no_grad():
        kink = _kinks(u, v, ok, du, dv, x, y, dhat.detach())
    gx = (ref[..., :, 1:] - ref[..., :, :-1]).abs().mean(1)
    gy = (ref[..., 1:, :] - ref[..., :-1, :]).abs().mean(1)
    sx = ((dhat[..., :, 1:] - dhat[..., :, :-1]).abs() * torch.exp(-gx)).sum() / (B * h * (w - 1))
    sy = ((dhat[..., 1:, :] - dhat[..., :-1, :]).abs() * torch.exp(-gy)).sum() / (B * (h - 1) * w)
    return LevelResult(e, valid, e_bound, sel, margin, kink, loss_q, Pl, sx + sy, N)


def _kinks(u, v, ok, du, dv, x, y, dhat):
    """(B,h,w) pixels p whose gradient is discontinuous within float32's rounding of the inputs
    it depends on: p's own warp (u or v) within twice its bound of a tap-cell edge, where the
    bilinear slope jumps; |x_c - y_c| at p within twice the sample bound of 0 (the L1 sign);
    a depth difference to a neighbour within 8 ulp of 0 (the smoothness sign)."""
    def near(t, dt):
        return (t - torch.round(t)).abs() < 2 * dt
    k = (ok & (near(u, du) | near(v, dv))).any(1)
    dy = (2 * (du + dv + 4 * EPS32))[:, :, None]
    k |= (ok[:, :, None] & ((x - y).abs() < dy)).any(2).any(1)
    tol = 8 * EPS32
    gx = (dhat[..., :, 1:] - dhat[..., :, :-1]).abs() < tol * (dhat[..., :, 1:].abs() + dhat[..., :, :-1].abs())
    gy = (dhat[..., 1:, :] - dhat[..., :-1, :]).abs() < tol * (dhat[..., 1:, :].abs() + dhat[..., :-1, :].abs())
    k[..., :, 1:] |= gx
    k[..., :, :-1] |= gx
    k[..., 1:, :] |= gy
    k[..., :-1, :] |= gy
    return k


def photo_loss(depths, imgs, proj_mats, dint, ratios, topk=1, smooth_weight=0.1, selected=None):
    """depths [(B,h_l,w_l)], imgs (B,V,3,H,W), proj_mats (B,S,levels,3,4), dint (B,) ->
    (L, [LevelResult]).  L = sum_l 2^(1-l) (P_l + smooth_weight S_l), differentiable in depths;
    `selected` is None or one (B,S,h,w) bool per level."""
    dint = torch.as_tensor(dint).reshape(-1).to(imgs.device)
    total, out = 0.0, []
    for l, d in enumerate(depths):
        r = level_loss(d, imgs, proj_mats[:, :, l], dint, float(ratios[l]), l, topk,
                       None if selected is None else selected[l])
        total = total + 2.0 ** (1 - l) * (r.P + smooth_weight * r.S)
        out.append(r)
    return total, out


def gradient(depths, imgs, proj_mats, dint, ratios, topk=1, smooth_weight=0.1, selected=None):
    """(L, [LevelResult], [dL/d depth_l]) in float64 (autograd of photo_loss)."""
    ds = [d.detach().double().requires_grad_(True) for d in depths]
    L, res = photo_loss(ds, imgs, proj_mats, dint, ratios, topk, smooth_weight, selected)
    grads = torch.autograd.grad(L, ds, allow_unused=True)
    grads = [torch.zeros_like(d) if g is None else g for d, g in zip(ds, grads)]
    return L.detach(), res, grads
