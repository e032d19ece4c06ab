"""Float64 reference of the convolution weight gradient (casmvs_conv3d_wgrad and
casmvs_conv3d_wgrad_det), for per-element checks; the companion of conv3d_fp64.conv3d_ref.

Plain torch only, like conv3d_fp64: the gradient of every tap is one contraction of a shifted
(strided) slice of the zero-padded input with the output gradient.  Tensors are channels-last:
x (B, D, h, w, Cin) the layer input, gy the gradient of the layer output (B, Do, ho, wo, Cout).
The result is in the packed tap-major layout of conv3d_fp64.pack_weight, (27, Cin, Cout):

    CONV            y[o] = sum_k xp[s*o + k] w[k]           dW[k] = sum_o xp[s*o + k]^T gy[o]
    CONV_TRANSPOSE  yp[2i + k] += x[i] w[k], y = yp[1:]     dW[k] = sum_i x[i]^T gyp[2i + k]

(xp, gyp: padded by one in front).  The library computes the transposed layer's gradient with
the roles of x and gy swapped, as (27, Cout, Cin): compare against wgrad_ref(...).transpose(1, 2).

Per-element bound of a kernel gradient dw against the float64 value dw64 (wgrad_bound_excess):
    |dw - dw64| <= eps * A + TINY,   A = wgrad_ref(|x|, |gy|)
A bounds every partial sum of any accumulation order, so eps is the accumulation's relative
error, as in conv3d_fp64.bound_excess.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .conv3d_fp64 import CONV, CONV_TRANSPOSE, TINY


def wgrad_ref(x, gy, kind, stride=1):
    """(27, Cin, Cout) float64 gradient of sum(y * gy) with respect to the packed weight of the
    layer y = conv(x): CONV is Conv3d(k3, pad 1, stride 1|2), CONV_TRANSPOSE
    ConvTranspose3d(k3, s2, p1, op1)."""
    x = x.to(torch.float64)
    gy = gy.to(device=x.device, dtype=torch.float64)
    taps = []
    if kind == CONV:
        B, Do, Ho, Wo, _ = gy.shape
        s = stride
        xp = F.pad(x, (0, 0, 1, 1, 1, 1, 1, 1))
        for kd in range(3):
            for kh in range(3):
                for kw in range(3):
                    xs = xp[:, kd:kd + s * (Do - 1) + 1:s, kh:kh + s * (Ho - 1) + 1:s,
                            kw:kw + s * (Wo - 1) + 1:s]
                    taps.append(torch.einsum("bdhwa,bdhwc->ac", xs, gy))
    elif kind == CONV_TRANSPOSE:
        B, D, H, W, _ = x.shape
        assert gy.shape[1:4] == (2 * D, 2 * H, 2 * W), (x.shape, gy.shape)
        gyp = F.pad(gy, (0, 0, 1, 1, 1, 1, 1, 1))
        for kd in range(3):
            for kh in range(3):
                for kw in range(3):
                    gs = gyp[:, kd:kd + 2 * D:2, kh:kh + 2 * H:2, kw:kw + 2 * W:2]
                    taps.append(torch.einsum("bdhwa,bdhwc->ac", x, gs))
    else:
        raise ValueError(f"no weight-gradient reference for kind {kind}")
    return torch.stack(taps)


def wgrad_magnitude(x, gy, kind, stride=1):
    """A = wgrad_ref(|x|, |gy|): bounds |partial sum| of every accumulation order."""
    return wgrad_ref(x.to(torch.float64).abs(), gy.to(torch.float64).abs(), kind, stride)


def wgrad_bound_excess(dw, dw64, A, eps):
    """Checks |dw - dw64| <= eps * A + TINY element by element.  dw (27, Ca, Cb) float32 (any
    device), dw64 and A float64 of the same shape.  Returns (ok, worst): worst is the smallest
    eps that would pass, max over elements of (|dw - dw64| - TINY)+ / A, with its location:
    dict(eps_needed, at=(tap, a, b), got, want, A)."""
    dw = dw.to(device=dw64.device, dtype=torch.float64)
    assert dw.shape == dw64.shape == A.shape, (dw.shape, dw64.shape, A.shape)
    over = ((dw - dw64).abs() - TINY).clamp_min(0)
    over = torch.where(torch.isnan(dw), torch.full_like(over, float("inf")), over)
    need = torch.where(over > 0, over / A, torch.zeros_like(over))     # over > 0 and A == 0: inf
    flat = int(torch.argmax(need.reshape(-1)).item())
    t, rest = divmod(flat, dw.shape[1] * dw.shape[2])
    a, b = divmod(rest, dw.shape[2])
    worst = dict(eps_needed=float(need[t, a, b]), at=(t, a, b), got=float(dw[t, a, b]),
                 want=float(dw64[t, a, b]), A=float(A[t, a, b]))
    return worst["eps_needed"] <= eps, worst
