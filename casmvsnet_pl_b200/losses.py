"""The training loss and depth metrics of the reference (losses.py, metrics.py) on
csrc/loss.cu, with no host synchronisation.

The reference computes `SmoothL1Loss(depth_pred_l[mask_l], depth_gt_l[mask_l]) * 2**(1-l)`
summed over the levels, and its metrics through the same boolean indexing; on CUDA every
`x[mask]` waits for the device to learn the output size.  Here one forward launch pair
produces the loss and level 0's metric sums in device memory, and the backward is one launch
whose gradients are bit-identical to autograd of the reference's expression.

    from casmvsnet_pl_b200.losses import loss_dict       # in place of the reference's losses.py
    loss = loss_dict['sl1'](levels=3)(results, depths, masks)

depth_metrics(pred, gt, mask) returns the (5,) device tensor
[sum |e|, #(|e| < 1), #(|e| < 2), #(|e| < 4), mask count]; accumulate it over batches and
divide once by the last entry (the mask-weighted means of train.py:157-163).
"""
from __future__ import annotations

import ctypes

import torch
from torch import nn

from . import _lib
from .ops import _ptr, _require_cuda, _stream, check


def _ptr_array(tensors):
    return (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def _prepare(preds, gts, masks):
    _require_cuda(*preds, *gts)
    B = preds[0].shape[0]
    p, g, m, hw = [], [], [], []
    for pl, gl, ml in zip(preds, gts, masks):
        if pl.dim() != 3 or pl.shape != gl.shape or pl.shape != ml.shape or pl.shape[0] != B:
            raise _lib.CasMVSError("sl1 loss expects (B,h,w) depth, target and mask per level, "
                                   f"got {tuple(pl.shape)}, {tuple(gl.shape)}, {tuple(ml.shape)}")
        if ml.dtype not in (torch.bool, torch.uint8) or ml.device != pl.device:
            raise _lib.CasMVSError("masks must be bool or uint8 tensors on the depth's device")
        p.append(pl.detach().contiguous())
        g.append(gl.detach().contiguous())
        m.append(ml.contiguous().view(torch.uint8))
        hw += [pl.shape[1], pl.shape[2]]
    return p, g, m, (ctypes.c_int * len(hw))(*hw), B


def _forward(preds, gts, masks):
    """-> loss (), metrics (5,), counts (levels,) int64, all on the device."""
    p, g, m, hw, B = _prepare(preds, gts, masks)
    dev = p[0].device
    lib = _lib.load()
    loss = torch.empty((), device=dev, dtype=torch.float32)
    metrics = torch.empty(5, device=dev, dtype=torch.float32)
    counts = torch.empty(len(p), device=dev, dtype=torch.int64)
    ws_bytes = lib.casmvs_sl1_loss_workspace_bytes()
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    with torch.cuda.device(dev):
        check(lib.casmvs_sl1_loss_fwd(_ptr_array(p), _ptr_array(g), _ptr_array(m), hw, B, len(p),
                                      _ptr(loss), _ptr(metrics), _ptr(counts), _ptr(ws), ws_bytes,
                                      _stream()), "sl1_loss_fwd")
    return loss, metrics, counts


class _SL1LossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, levels, *tensors):
        preds, gts, masks = tensors[:levels], tensors[levels:2 * levels], tensors[2 * levels:]
        loss, metrics, counts = _forward(preds, gts, masks)
        ctx.save_for_backward(*tensors, counts)
        ctx.levels = levels
        ctx.mark_non_differentiable(metrics)
        return loss, metrics

    @staticmethod
    def backward(ctx, grad_loss, _grad_metrics):
        L = ctx.levels
        *tensors, counts = ctx.saved_tensors
        p, g, m, hw, B = _prepare(tensors[:L], tensors[L:2 * L], tensors[2 * L:])
        grads = [torch.empty_like(t) for t in p]
        go = grad_loss.detach().to(torch.float32).contiguous()
        with torch.cuda.device(p[0].device):
            check(_lib.load().casmvs_sl1_loss_bwd(_ptr_array(p), _ptr_array(g), _ptr_array(m), hw, B,
                                                  L, _ptr(counts), _ptr(go), _ptr_array(grads),
                                                  _stream()), "sl1_loss_bwd")
        return (None, *[gr if ctx.needs_input_grad[1 + i] else None for i, gr in enumerate(grads)],
                *([None] * (2 * L)))


def sl1_loss_and_metrics(inputs, targets, masks, levels=3):
    """(loss (), metrics (5,)) of the reference's SL1Loss and level-0 metrics in one launch pair.
    inputs: {'depth_l'}, targets / masks: {'level_l'} (datasets/dtu.py sample layout)."""
    preds = [inputs[f"depth_{l}"] for l in range(levels)]
    gts = [targets[f"level_{l}"] for l in range(levels)]
    ms = [masks[f"level_{l}"] for l in range(levels)]
    return _SL1LossFn.apply(levels, *preds, *gts, *ms)


class SL1Loss(nn.Module):
    """losses.py:4-17: sum_l 2^(1-l) * SmoothL1Loss(reduction='mean') over mask_l."""

    def __init__(self, levels=3):
        super().__init__()
        self.levels = levels

    def forward(self, inputs, targets, masks):
        return sl1_loss_and_metrics(inputs, targets, masks, self.levels)[0]


loss_dict = {"sl1": SL1Loss}


def depth_metrics(pred, gt, mask):
    """(5,) float32 device tensor [sum |e|, #(|e| < 1), #(|e| < 2), #(|e| < 4), n] of the masked
    errors e = pred - gt (metrics.py: abs_error and acc_threshold at 1, 2, 4, summed)."""
    with torch.no_grad():
        return _forward([pred], [gt], [mask])[1]


# ------------------------------------------------------------------ photometric (csrc/photo_loss.cu)
def _photo_inputs(depths, imgs, proj_mats, depth_interval, interval_ratios, levels):
    _require_cuda(imgs, proj_mats, *depths)
    if imgs.dim() != 5 or imgs.shape[2] != 3:
        raise _lib.CasMVSError(f"photo loss expects imgs (B,V,3,H,W), got {tuple(imgs.shape)}")
    B, V, _, H, W = imgs.shape
    if tuple(proj_mats.shape) != (B, V - 1, levels, 3, 4):
        raise _lib.CasMVSError(f"photo loss expects proj_mats {(B, V - 1, levels, 3, 4)}, "
                               f"got {tuple(proj_mats.shape)}")
    for l, d in enumerate(depths):
        if tuple(d.shape) != (B, H >> l, W >> l) or d.device != imgs.device or d.dtype != torch.float32:
            raise _lib.CasMVSError(f"depth_{l} must be float32 {(B, H >> l, W >> l)} on the images' device, "
                                   f"got {tuple(d.shape)}")
    if len(interval_ratios) < levels:
        raise _lib.CasMVSError(f"{levels} levels need {levels} interval ratios")
    dint = torch.as_tensor(depth_interval, dtype=torch.float32, device=imgs.device).reshape(-1)
    if dint.numel() == 1 and B > 1:
        dint = dint.expand(B)
    if dint.numel() != B:
        raise _lib.CasMVSError(f"depth_interval must have one value per sample, got {dint.numel()}")
    ratios = (ctypes.c_float * levels)(*[float(r) for r in interval_ratios[:levels]])
    return (imgs.detach().float().contiguous(), proj_mats.detach().float().contiguous(),
            dint.contiguous(), [d.detach().contiguous() for d in depths], ratios, (B, V, H, W))


class _PhotoLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, levels, topk, smooth_weight, interval_ratios, debug_maps, imgs, proj_mats,
                depth_interval, *depths):
        im, pm, dint, ds, ratios, (B, V, H, W) = _photo_inputs(depths, imgs, proj_mats, depth_interval,
                                                               interval_ratios, levels)
        dev = im.device
        lib = _lib.load()
        loss = torch.empty((), device=dev, dtype=torch.float32)
        stats = torch.empty(levels, 3, device=dev, dtype=torch.float32)
        counts = torch.empty(levels, device=dev, dtype=torch.int64)
        sel = [torch.empty(d.shape, device=dev, dtype=torch.int16) for d in ds]
        ws_bytes = lib.casmvs_photo_loss_workspace_bytes(B, H, W, levels)
        ws = torch.empty(max(ws_bytes, 1), device=dev, dtype=torch.uint8)
        dbg_e = dbg_valid = dbg_lossq = None
        if debug_maps is not None:
            dbg_e = [torch.empty(B, V - 1, *d.shape[1:], device=dev) for d in ds]
            dbg_valid = [torch.empty(d.shape, device=dev, dtype=torch.int16) for d in ds]
            dbg_lossq = [torch.empty(d.shape, device=dev) for d in ds]
        opt = lambda ts: None if ts is None else _ptr_array(ts)   # noqa: E731
        with torch.cuda.device(dev):
            check(lib.casmvs_photo_loss_fwd(_ptr(im), _ptr(pm), _ptr(dint), _ptr_array(ds), ratios, B, V,
                                            H, W, levels, topk, smooth_weight, _ptr_array(sel),
                                            _ptr(loss), _ptr(stats), _ptr(counts), opt(dbg_e),
                                            opt(dbg_valid), opt(dbg_lossq), _ptr(ws), ws_bytes,
                                            _stream()), "photo_loss_fwd")
        ctx.save_for_backward(im, pm, dint, counts, *ds, *sel)
        ctx.args = (levels, topk, smooth_weight, ratios, (B, V, H, W))
        ctx.mark_non_differentiable(stats)
        if debug_maps is not None:
            debug_maps += [{"e": e, "valid": _bits(v, V - 1), "selected": _bits(s, V - 1), "loss_q": q}
                           for e, v, s, q in zip(dbg_e, dbg_valid, sel, dbg_lossq)]
        return loss, stats

    @staticmethod
    def backward(ctx, grad_loss, _grad_stats):
        levels, topk, smooth_weight, ratios, (B, V, H, W) = ctx.args
        im, pm, dint, counts, *rest = ctx.saved_tensors
        ds, sel = rest[:levels], rest[levels:]
        grads = [torch.empty_like(d) for d in ds]
        go = grad_loss.detach().to(torch.float32).contiguous()
        with torch.cuda.device(im.device):
            check(_lib.load().casmvs_photo_loss_bwd(_ptr(im), _ptr(pm), _ptr(dint), _ptr_array(ds), ratios,
                                                    B, V, H, W, levels, topk, smooth_weight,
                                                    _ptr_array(sel), _ptr(counts), _ptr(go),
                                                    _ptr_array(grads), _stream()), "photo_loss_bwd")
        return (None,) * 8 + tuple(grads)


def _bits(mask16, S):
    """(B,h,w) int16 bit masks -> (B,S,h,w) bool, bit s -> [:, s]."""
    m = mask16.to(torch.int32) & 0xFFFF
    return torch.stack([(m >> s) & 1 for s in range(S)], 1).bool()


def photo_loss(results, imgs, proj_mats, depth_interval, interval_ratios, levels=3, topk=1,
               smooth_weight=0.01, debug=False):
    """Self-supervised photometric loss of depth maps `results['depth_l']` (csrc/photo_loss.cu
    states the rule): each source image is warped into the reference view with the predicted
    depth, the 3x3 SSIM + L1 errors of the `topk` best sources per pixel are averaged, and an
    edge-aware smoothness of depth in hypothesis spacings is added with weight smooth_weight.

    imgs (B,V,3,H,W) normalised network input, proj_mats (B,V-1,levels,3,4) as the model takes,
    depth_interval (B,1) or (B,), interval_ratios one per level.  Returns (loss (), stats
    (levels,3) = [P_l, S_l, N_l]), device tensors, with no host synchronisation; only the depth
    maps get a gradient.  debug=True adds a third value, per level {e (B,S,h,w) NaN where
    invalid, valid (B,S,h,w) bool, selected (B,S,h,w) bool, loss_q (B,h,w) NaN where no source
    is valid}."""
    depths = [results[f"depth_{l}"] for l in range(levels)]
    maps = [] if debug else None
    loss, stats = _PhotoLossFn.apply(levels, topk, float(smooth_weight), list(interval_ratios), maps,
                                     imgs, proj_mats, depth_interval, *depths)
    return (loss, stats, maps) if debug else (loss, stats)
