"""Differentiable wrappers of the hot-path kernels (SURVEY.md 8 f-1): what the reference's
training step (train.py:99-127: forward, SL1 loss on depth_l, backward) needs.

  WarpCostFn   K1: d(cost volume)/d(features) by casmvs_warp_cost_bwd (grid_sample's backward
               chained with the variance / group-wise-correlation reduction).  Hypotheses are
               detached in the reference (models/mvsnet.py:231), projections are data.
  Conv3dFn     K2: the raw 3x3x3 (transposed) convolution; data gradient = one of the forward
               kernels with re-arranged weights, weight gradient = casmvs_conv3d_wgrad.  The
               norm-act that follows it in training mode is batch-statistics ABN
               (casmvsnet_pl_b200.norm_act: F.batch_norm + leaky_relu, torch autograd).
  RegressFn    K3: d(depth)/d(logits); confidence is computed under no_grad (mvsnet.py:179).
  Upsample2xFn FeatureNet's bilinear x2 upsample (align_corners=True): ATen's forward, backward
               by casmvs_upsample2x_bilinear_bwd.

With torch.use_deterministic_algorithms(True) the backward ops run the deterministic entries
(casmvs_warp_cost_bwd_det, casmvs_conv3d_wgrad_det, casmvs_upsample2x_bilinear_bwd): a training
step is then the same bits for the same inputs.  `deterministic()` below is the one place that
decides; without it every op runs exactly as before.
"""
from __future__ import annotations

import ctypes

import torch
import torch.nn.functional as F

from . import _lib, ops
from .ops import CONV, CONV_TRANSPOSE, FP32, NCHW, NHWC, TF32, _ptr, _stream, check


def deterministic():
    """torch's switch: the deterministic backward kernels run when it is on."""
    return torch.are_deterministic_algorithms_enabled()


def _workspace(nbytes, device):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


def _dense_ndhwc(x):
    """logical (B,C,D,h,w) -> dense (B,D,h,w,C)."""
    return ops.volume_storage(x)


class WarpCostFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feats, proj_mats, depth_values, num_groups):
        f = feats.detach()
        cost = ops.warp_cost(f, proj_mats, depth_values, num_groups, NHWC)
        B, V, C, h, w = f.shape
        f_cl = f.permute(0, 1, 3, 4, 2).contiguous()          # (B,V,h,w,C); no copy if channels-last
        ctx.save_for_backward(f_cl, proj_mats.contiguous(), depth_values.contiguous())
        ctx.G = num_groups
        return cost

    @staticmethod
    def backward(ctx, gcost):
        f_cl, proj, dv = ctx.saved_tensors
        B, V, h, w, C = f_cl.shape
        D = dv.shape[1]
        g = _dense_ndhwc(gcost)
        lib = _lib.load()
        with torch.cuda.device(f_cl.device):
            if deterministic():
                gf = torch.empty_like(f_cl)
                ws = _workspace(lib.casmvs_warp_cost_bwd_det_workspace_bytes(B, V, C, D, h, w), f_cl.device)
                check(lib.casmvs_warp_cost_bwd_det(_ptr(f_cl), _ptr(proj), _ptr(dv), _ptr(g), _ptr(gf),
                                                   B, V, C, D, h, w, ctx.G, _ptr(ws), ws.numel(),
                                                   _stream()), "warp_cost_bwd_det")
            else:
                gf = torch.zeros_like(f_cl)
                check(lib.casmvs_warp_cost_bwd(_ptr(f_cl), _ptr(proj), _ptr(dv), _ptr(g), _ptr(gf),
                                               B, V, C, D, h, w, ctx.G, _stream()), "warp_cost_bwd")
        return gf.permute(0, 1, 4, 2, 3), None, None, None


def _tf32_operand(x, cin, cout, kind, stride, precision):
    """The activation operand as the layer's kernel should read it.  A tensor-core kernel reads
    only the top 19 bits of an fp32 value, which biases every product toward zero by about
    2^-11 of its size.  The inference path stores its activations TF32-rounded for that reason;
    here the torch norm-act output, the cost volume and the gradients are full fp32.  So where a
    tensor-core kernel runs, x is RNA-rounded into a new buffer (x itself may be the previous
    layer's activation, or a gradient autograd also sends to a skip branch).  A TF32-exact value
    is unchanged.  The CUDA-core fallback multiplies fp32 operands exactly and reads x as is."""
    if (precision & 0xff) != TF32 or not ops.conv3d_tensor_core(cin, cout, kind, stride):
        return x
    r = _dense_ndhwc(x).clone()
    B, D, h, w, C = r.shape
    ops.bias_lrelu_(r.view(B * D, h, w, C).permute(0, 3, 1, 2), torch.zeros(C, device=r.device),
                    1.0, round_tf32=True)
    return ops.as_volume_view(r)


def _raw_conv(x, weight_torch, kind, stride, precision):
    """-> (y, the operand the kernel read: x, or x rounded to TF32 by _tf32_operand)."""
    cin, cout = (weight_torch.shape[1], weight_torch.shape[0]) if kind == CONV else \
        (weight_torch.shape[0], weight_torch.shape[1])
    x = _tf32_operand(x, cin, cout, kind, stride, precision)
    wp = ops.pack_conv3d_weight(weight_torch, kind)
    y = ops.conv3d(x, wp, cin, cout, None, None, 1.0, None, kind, stride, precision)
    ops.release_weight_images(wp)          # one-shot weights: do not let operand images pile up
    return y, x


class Conv3dFn(torch.autograd.Function):
    """y = Conv3d(k3, pad 1, stride 1|2)(x) or ConvTranspose3d(k3, s2, p1, op1)(x), no bias."""

    @staticmethod
    def forward(ctx, x, weight, kind, stride, precision):
        wd = weight.detach()
        # the weight gradient takes the operand the kernel read: the function it computed
        y, xd = _raw_conv(x.detach(), wd, kind, stride, precision)
        ctx.save_for_backward(xd, wd)
        ctx.cfg = (kind, stride, precision)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w = ctx.saved_tensors
        kind, stride, precision = ctx.cfg
        gx = gw = None
        gyd = _dense_ndhwc(gy)                                  # (B,Do,ho,wo,Cout)
        gy_l = ops.as_volume_view(gyd)
        xs = _dense_ndhwc(x)
        B, Di, hi, wi, cin = xs.shape
        _, Do, ho, wo, cout = gyd.shape
        if ctx.needs_input_grad[0]:
            if kind == CONV and stride == 1:
                # adjoint of a stride-1 correlation: correlate with the flipped kernel, channels swapped
                wt = w.flip(2, 3, 4).transpose(0, 1).contiguous()            # (Cin,Cout,3,3,3)
                g_in = gy_l
                if cout % 4:                                                 # prob head: Cout = 1
                    pad = 4 - cout % 4
                    g_in = ops.as_volume_view(torch.nn.functional.pad(gyd, (0, pad)))
                    wt = torch.nn.functional.pad(wt, (0, 0, 0, 0, 0, 0, 0, pad))
                gx, _ = _raw_conv(g_in, wt, CONV, 1, precision)
            elif kind == CONV:
                # conv(k3,s2,p1) on even dims: its adjoint is ConvTranspose3d(k3,s2,p1,op1) with
                # the SAME weight tensor read as (in = Cout, out = Cin)
                gx, _ = _raw_conv(gy_l, w, CONV_TRANSPOSE, 2, precision)
            else:
                # adjoint of the transposed conv: Conv3d(k3,s2,p1), weight read as (out=Cin, in=Cout)
                gx, _ = _raw_conv(gy_l, w, CONV, 2, precision)
        if ctx.needs_input_grad[1]:
            with torch.cuda.device(x.device):
                if kind == CONV:
                    dw = _wgrad(xs, gyd, B, cin, cout, (Di, hi, wi), (Do, ho, wo), stride)
                    gw = dw.view(3, 3, 3, cin, cout).permute(4, 3, 0, 1, 2).contiguous()
                else:
                    # y[2i-1+k] += x[i] w[k]: the output gradient plays the strided input
                    dw = _wgrad(gyd, xs, B, cout, cin, (Do, ho, wo), (Di, hi, wi), 2)
                    gw = dw.view(3, 3, 3, cout, cin).permute(4, 3, 0, 1, 2).contiguous()
        return gx, gw, None, None, None


def _wgrad(x, gy, B, ca, cb, xdims, ydims, stride):
    """(27, ca, cb) weight gradient of casmvs_conv3d_wgrad, or of its deterministic variant."""
    lib = _lib.load()
    if deterministic():
        dw = torch.empty(27, ca, cb, device=x.device, dtype=torch.float32)
        ws = _workspace(lib.casmvs_conv3d_wgrad_det_workspace_bytes(B, ca, cb, *ydims), x.device)
        check(lib.casmvs_conv3d_wgrad_det(_ptr(x), _ptr(gy), _ptr(dw), B, ca, cb, *xdims, *ydims, stride,
                                          _ptr(ws), ws.numel(), _stream()), "conv3d_wgrad_det")
    else:
        dw = torch.zeros(27, ca, cb, device=x.device, dtype=torch.float32)
        check(lib.casmvs_conv3d_wgrad(_ptr(x), _ptr(gy), _ptr(dw), B, ca, cb, *xdims, *ydims, stride,
                                      _stream()), "conv3d_wgrad")
    return dw


def _regress_fwd(ctx, logits, depth_values, inverse):
    lg = logits.detach().contiguous()
    dv = depth_values.contiguous()
    depth, conf, _, _ = ops.regress(lg, dv, inverse=inverse)
    ctx.save_for_backward(lg, dv)
    ctx.mark_non_differentiable(conf)
    return depth, conf


def _regress_bwd(ctx, gdepth, inverse):
    lg, dv = ctx.saved_tensors
    B, D, h, w = lg.shape
    out = torch.empty_like(lg)
    with torch.cuda.device(lg.device):
        flags = int(dv.dim() == 1) | (ops.INVERSE_DEPTH if inverse else 0)
        check(_lib.load().casmvs_regress_bwd(_ptr(lg), _ptr(dv), flags,
                                             _ptr(gdepth.contiguous()), _ptr(out), B, D, h, w,
                                             _stream()), "regress_bwd")
    return out, None


class RegressFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, depth_values):
        return _regress_fwd(ctx, logits, depth_values, False)

    @staticmethod
    def backward(ctx, gdepth, _gconf):
        return _regress_bwd(ctx, gdepth, False)


class RegressInverseFn(torch.autograd.Function):
    """RegressFn in 1/depth: depth = 1/sum_d p_d/dv_d, d depth/d l_d = -depth^2 p_d (1/dv_d - 1/depth)."""

    @staticmethod
    def forward(ctx, logits, depth_values):
        return _regress_fwd(ctx, logits, depth_values, True)

    @staticmethod
    def backward(ctx, gdepth, _gconf):
        return _regress_bwd(ctx, gdepth, True)


class RegressSpreadFn(torch.autograd.Function):
    """RegressFn that also returns the adaptive mode's spread (README "Adaptive depth ranges"),
    non-differentiable like the confidence; depth's gradient is RegressFn's."""

    @staticmethod
    def forward(ctx, logits, depth_values):
        lg = logits.detach().contiguous()
        dv = depth_values.contiguous()
        depth, conf, _, _, spread = ops.regress(lg, dv, want_spread=True)
        ctx.save_for_backward(lg, dv)
        ctx.mark_non_differentiable(conf, spread)
        return depth, conf, spread

    @staticmethod
    def backward(ctx, gdepth, _gconf, _gspread):
        return _regress_bwd(ctx, gdepth, False)


class Upsample2xFn(torch.autograd.Function):
    """F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True) of a CUDA fp32
    (N,C,h,w) tensor, NCHW or channels-last: ATen's forward, the gather backward."""

    @staticmethod
    def forward(ctx, x):
        return F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)

    @staticmethod
    def backward(ctx, gy):
        N, C, H, W = gy.shape
        nhwc = gy.is_contiguous(memory_format=torch.channels_last) and not gy.is_contiguous()
        g = gy if nhwc else gy.contiguous()
        gx = torch.empty(N, C, H // 2, W // 2, device=gy.device, dtype=torch.float32,
                         memory_format=torch.channels_last if nhwc else torch.contiguous_format)
        with torch.cuda.device(gy.device):
            check(_lib.load().casmvs_upsample2x_bilinear_bwd(_ptr(g), _ptr(gx), N, C, H // 2, W // 2,
                                                             NHWC if nhwc else NCHW, _stream()),
                  "upsample2x_bilinear_bwd")
        return gx


def upsample2x(x):
    """FeatureNet's x2 bilinear upsample (align_corners=True).  torch's own backward scatters
    with atomics, and raises under torch.use_deterministic_algorithms(True): a CUDA fp32 input
    then takes Upsample2xFn's gather backward instead."""
    if deterministic() and x.is_cuda and x.dtype == torch.float32 and torch.is_grad_enabled():
        return Upsample2xFn.apply(x)
    return F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)


def conv3d(x, weight, kind=CONV, stride=1, precision=FP32):
    return Conv3dFn.apply(x, weight, kind, stride, precision)


def warp_cost(feats, proj_mats, depth_values, num_groups=1):
    return WarpCostFn.apply(feats, proj_mats, depth_values, num_groups)


def regress(logits, depth_values, inverse=False, want_spread=False):
    """inverse=True: the inverse-depth regression, depth = 1/sum_d p_d/depth_values_d.
    want_spread=True: (depth, confidence, spread), the spread without a gradient."""
    if want_spread:
        if inverse:
            raise _lib.CasMVSError("regress: want_spread is the adaptive mode's, not the inverse mode's")
        return RegressSpreadFn.apply(logits, depth_values)
    return (RegressInverseFn if inverse else RegressFn).apply(logits, depth_values)
