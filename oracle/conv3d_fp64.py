"""Float64 reference of the engine's convolution layers (K2), for per-element checks.

Plain torch only (no casmvsnet_pl_b200 import, no F.conv* / cuDNN): every layer is a sum over
its taps of a shifted (strided) slice of the zero-padded input contracted with that tap's weight
matrix, or for the transposed convolution a scatter of x[i] w[k] into a padded output.  The same
functions run on the CPU and, for the large shapes, on the GPU: the arithmetic is float64
either way, so where it runs changes only float64 rounding.

Tensors are channels-last, like the engine's volumes: x (B, D, h, w, Cin); weights are in the
packed tap-major layout of casmvs_pack_conv3d_weights, (27, Cin, Cout) with tap =
(kd*3 + kh)*3 + kw unflipped (for CONV_TRANSPOSE the torch (Cin, Cout, 3, 3, 3) weight's taps),
or (25, Cin, Cout) with tap = kh*5 + kw for the 5x5 stride-2 Conv2d.

Per-element bound of a kernel output y against the float64 value y64 (bound_excess):
    |y - y64| <= eps * A + r * |y64| + tiny
A = |scale| * conv3d_ref(|x|, |w|) bounds every partial sum of the accumulation, so eps is the
accumulator's relative error; r = 2^-11 where the output is stored TF32-rounded (half an ulp
of a 10-bit mantissa), 0 otherwise; tiny = 2^-22 * (|shift| + |skip|) covers the fp32 roundings
of the epilogue additions, which A does not bound.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

# layer kinds: the library's casmvs_conv_kind values, plus the 5x5 stride-2 Conv2d of FeatureNet
CONV, CONV_TRANSPOSE, CONV_PLANAR, CONV5X5_S2 = 0, 1, 2, 3

R_TF32 = 2.0 ** -11          # relative rounding error of a TF32-rounded store
EPI_REL = 2.0 ** -22         # epilogue roundings relative to |shift| + |skip|
TINY = 2.0 ** -120           # absolute floor (outputs that are exactly zero in float64)


def pack_weight(w_torch, kind):
    """torch weight -> packed (taps, Cin, Cout) float64, the layout casmvs_pack_conv3d_weights
    writes: Conv3d (Cout,Cin,3,3,3), ConvTranspose3d (Cin,Cout,3,3,3), planar Conv2d
    (Cout,Cin,3,3) -> centre plane of 27 taps, 5x5 Conv2d (Cout,Cin,5,5) -> 25 taps."""
    w = w_torch.detach().to(torch.float64)
    if kind == CONV:
        return w.permute(2, 3, 4, 1, 0).reshape(27, w.shape[1], w.shape[0]).contiguous()
    if kind == CONV_TRANSPOSE:
        return w.permute(2, 3, 4, 0, 1).reshape(27, w.shape[0], w.shape[1]).contiguous()
    if kind == CONV_PLANAR:
        out = w.new_zeros(27, w.shape[1], w.shape[0])
        out[9:18] = w.permute(2, 3, 1, 0).reshape(9, w.shape[1], w.shape[0])
        return out
    if kind == CONV5X5_S2:
        return w.permute(2, 3, 1, 0).reshape(25, w.shape[1], w.shape[0]).contiguous()
    raise ValueError(f"unknown kind {kind}")


def out_dims(kind, stride, D, h, w):
    if kind == CONV_TRANSPOSE:
        return 2 * D, 2 * h, 2 * w
    if kind == CONV5X5_S2:
        return D, (h - 1) // 2 + 1, (w - 1) // 2 + 1
    if kind == CONV_PLANAR:
        return D, h, w
    return (D - 1) // stride + 1, (h - 1) // stride + 1, (w - 1) // stride + 1


def _tap(xs, wk):
    return torch.einsum("bdhwc,co->bdhwo", xs, wk)


def conv3d_ref(x, w, kind, stride=1):
    """Raw convolution (no epilogue) of channels-last x (B,D,h,w,Cin) with packed w, float64.
    CONV: Conv3d(k3, pad 1, stride 1|2); CONV_TRANSPOSE: ConvTranspose3d(k3, s2, p1, op1);
    CONV_PLANAR: 1x3x3, pad (0,1,1); CONV5X5_S2: 5x5 stride-2 pad-2 Conv2d of every (h, w)
    image of the (D = views, h, w) volume."""
    x = x.to(torch.float64)
    w = w.to(device=x.device, dtype=torch.float64)
    B, D, H, W, _ = x.shape
    cout = w.shape[-1]
    Do, Ho, Wo = out_dims(kind, stride, D, H, W)
    if kind == CONV_TRANSPOSE:
        # y[2i - 1 + k] += x[i] w[k]: padded output index 2i + k, cropped to 1 .. 2n
        yp = x.new_zeros(B, 2 * D + 1, 2 * H + 1, 2 * W + 1, cout)
        for kd in range(3):
            for kh in range(3):
                for kw in range(3):
                    yp[:, kd:kd + 2 * D:2, kh:kh + 2 * H:2, kw:kw + 2 * W:2] += \
                        _tap(x, w[(kd * 3 + kh) * 3 + kw])
        return yp[:, 1:2 * D + 1, 1:2 * H + 1, 1:2 * W + 1]
    y = x.new_zeros(B, Do, Ho, Wo, cout)
    if kind == CONV5X5_S2:
        xp = F.pad(x, (0, 0, 2, 2, 2, 2))
        for kh in range(5):
            for kw in range(5):
                y += _tap(xp[:, :, kh:kh + 2 * (Ho - 1) + 1:2, kw:kw + 2 * (Wo - 1) + 1:2],
                          w[kh * 5 + kw])
        return y
    if kind == CONV_PLANAR:
        xp = F.pad(x, (0, 0, 1, 1, 1, 1))
        for kh in range(3):
            for kw in range(3):
                y += _tap(xp[:, :, kh:kh + Ho, kw:kw + Wo], w[9 + kh * 3 + kw])
        return y
    s = stride
    xp = F.pad(x, (0, 0, 1, 1, 1, 1, 1, 1))
    for kd in range(3):
        for kh in range(3):
            for kw in range(3):
                y += _tap(xp[:, kd:kd + s * (Do - 1) + 1:s, kh:kh + s * (Ho - 1) + 1:s,
                             kw:kw + s * (Wo - 1) + 1:s], w[(kd * 3 + kh) * 3 + kw])
    return y


def dgrad_ref(gy, w, kind, stride, in_dims):
    """Float64 data gradient of the raw layer: the vector-Jacobian product of conv3d_ref with
    packed w at an input of dims in_dims = (D, h, w), applied to gy (B, Do, ho, wo, Cout), by
    torch.autograd in float64 -> (B, D, h, w, Cin).  No flipped, transposed or padded weight is
    built by hand, so a mistake in such a construction elsewhere cannot cancel here.  The map
    is linear, so dgrad_ref(|gy|, |w|) is the magnitude of the per-element bound."""
    gy = gy.to(torch.float64)
    w = w.to(device=gy.device, dtype=torch.float64)
    x = gy.new_zeros(gy.shape[0], *in_dims, w.shape[-2], requires_grad=True)
    with torch.enable_grad():
        y = conv3d_ref(x, w, kind, stride)
        assert y.shape == gy.shape, (y.shape, gy.shape)
        (gx,) = torch.autograd.grad(y, x, gy)
    return gx


def operand_bias(y, y64):
    """sum (y - y64) sign(y64) / sum |y64|: the mean relative error of y in the direction of
    y64.  About 0 where the operands were rounded to nearest; about -2^-11 (toward zero) where
    the low 13 mantissa bits of a non-TF32 operand were dropped."""
    y = y.to(device=y64.device, dtype=torch.float64)
    return float(((y - y64) * torch.sign(y64)).sum() / y64.abs().sum().clamp_min(TINY))


def tf32_trunc(t):
    """A float32 tensor with its low 13 mantissa bits cleared (round toward zero to TF32)."""
    assert t.dtype == torch.float32
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def epilogue(acc, scale=None, shift=None, slope=1.0, skip=None):
    """lrelu(scale * acc + shift, slope) + skip, float64, per output channel (last dim)."""
    v = acc
    if scale is not None:
        v = v * scale.to(device=v.device, dtype=torch.float64)
    if shift is not None:
        v = v + shift.to(device=v.device, dtype=torch.float64)
    v = torch.where(v >= 0, v, v * slope)
    if skip is not None:
        v = v + skip.to(device=v.device, dtype=torch.float64)
    return v


def magnitude(x, w, kind, stride=1, scale=None):
    """A = |scale| * conv3d_ref(|x|, |w|): bounds |scale * partial sum| of every accumulation
    order, the scale of the per-element tolerance."""
    a = conv3d_ref(x.to(torch.float64).abs(), w.to(torch.float64).abs(), kind, stride)
    if scale is not None:
        a = a * scale.to(device=a.device, dtype=torch.float64).abs()
    return a


def epilogue_magnitude(shape_like, shift=None, skip=None):
    """|shift| + |skip| broadcast to the output: the epilogue addends A does not bound."""
    m = torch.zeros((), dtype=torch.float64, device=shape_like.device)
    if shift is not None:
        m = m + shift.to(device=shape_like.device, dtype=torch.float64).abs()
    if skip is not None:
        m = m + skip.to(device=shape_like.device, dtype=torch.float64).abs()
    return m


def tf32_rna(t):
    """Exact emulation of cvt.rna.tf32.f32: round a float32 tensor to a 10-bit mantissa, to
    nearest with ties away from zero, on the int32 bits (sign-magnitude: adding half an ulp of
    the magnitude rounds both signs away).  A finite value that rounds past the largest TF32
    becomes infinity; infinities and NaNs are returned unchanged."""
    assert t.dtype == torch.float32
    bits = t.contiguous().view(torch.int32)
    rounded = (bits + 0x1000) & ~0x1FFF
    return torch.where(torch.isfinite(t), rounded, bits).view(torch.float32)


def to_blocked(x):
    """(B, D, h, w, C) channels-last -> contiguous (B, C/4, D, h, w, 4)."""
    B, D, h, w, C = x.shape
    return x.reshape(B, D, h, w, C // 4, 4).permute(0, 4, 1, 2, 3, 5).contiguous()


def from_blocked(xb):
    """(B, C/4, D, h, w, 4) -> contiguous (B, D, h, w, C)."""
    B, Q, D, h, w, _ = xb.shape
    return xb.permute(0, 2, 3, 4, 1, 5).reshape(B, D, h, w, 4 * Q)


def bound_excess(y, y64, A, eps, r=0.0, extra=None):
    """Checks |y - y64| <= eps * A + r * |y64| + EPI_REL * extra + TINY element by element.

    y (B,D,h,w,C) float32 (any device), y64 / A float64 of the same shape, extra = |shift| +
    |skip| (broadcastable) or None.  Returns (ok, worst): worst is the smallest eps that would
    pass, i.e. max over voxels of (|y - y64| - r|y64| - EPI_REL*extra - TINY)+ / A, with its
    location: dict(eps_needed, at=(b, d, h, w, c), h16, w8, slice, got, want, A)."""
    y = y.to(device=y64.device, dtype=torch.float64)
    assert y.shape == y64.shape == A.shape, (y.shape, y64.shape, A.shape)
    slack = r * y64.abs() + TINY
    if extra is not None:
        slack = slack + EPI_REL * extra
    over = ((y - y64).abs() - slack).clamp_min(0)
    over = torch.where(torch.isnan(y), torch.full_like(over, float("inf")), over)
    need = torch.where(over > 0, over / A, torch.zeros_like(over))     # over > 0 and A == 0: inf
    flat = int(torch.argmax(need.reshape(-1)).item())
    idx = []
    for n in reversed(y.shape):
        idx.append(flat % n)
        flat //= n
    b, d, h, w, c = reversed(idx)
    worst = dict(eps_needed=float(need[b, d, h, w, c]), at=(b, d, h, w, c), h16=h % 16, w8=w % 8,
                 slice=d, got=float(y[b, d, h, w, c]), want=float(y64[b, d, h, w, c]),
                 A=float(A[b, d, h, w, c]))
    return worst["eps_needed"] <= eps, worst
