"""Training panels on the GPU (csrc/visual.cu; numpy restatement in oracle/visual_oracle.py,
byte for byte): the original project's utils/visualization.py and the image it logs to
TensorBoard at batch 0 of every epoch.

    strip = training_panel(img, depth_gt, depth_pred, conf, mask)   # (H, 4W, 3) uint8
    x = visualize_depth(depth)                                       # (3, H, W) float32
    x = visualize_prob(prob)                                         # (3, H, W) float32

training_panel draws the un-normalised reference image, visualize_depth(depth_gt),
visualize_depth(depth_pred * mask) and visualize_prob(conf * mask) side by side: the bytes that
TensorBoard stores for the original's add_images('train/image_GT_pred_prob', stack).  Depth goes
through cv2's JET colour map, confidence through BONE, and as in the original both show blue and
red swapped (cv2's BGR read as RGB).  A depth map with no positive value, where the original
raises, is drawn in the colour of grey level 0.  Everything stays on the device; nothing
synchronises the host.
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _check(name, t, dtype, shape, device):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor")
    if t.dtype not in dtype:
        raise ValueError(f"{name} must be {' or '.join(str(d) for d in dtype)}, got {t.dtype}")
    if tuple(t.shape) != shape:
        raise ValueError(f"{name} must have shape {shape}, got {tuple(t.shape)}")
    if device is not None and t.device != device:
        raise ValueError(f"{name} is on {t.device}, the other inputs on {device}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    return t


def _map_shape(name, t):
    if not torch.is_tensor(t) or t.dim() != 2 or min(t.shape) < 1:
        raise ValueError(f"{name} must be a non-empty (H, W) tensor")
    return tuple(t.shape)


def _panels(img, depth_gt, depth_pred, conf, mask, shape, device):
    """Launches the kernel pair on the current stream -> (H, n*W, 3) uint8."""
    H, W = shape
    n = sum(t is not None for t in (img, depth_gt, depth_pred, conf))
    with torch.cuda.device(device):
        out = torch.empty(H, n * W, 3, dtype=torch.uint8, device=device)
        ws = torch.empty(_lib.VISUAL_WORKSPACE_BYTES // 4, dtype=torch.float32, device=device)
        _lib.check(_lib.load().casmvs_visual_panels(
            _ptr(img), _ptr(depth_gt), _ptr(depth_pred), _ptr(conf), _ptr(mask), H, W, _ptr(out),
            _ptr(ws), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "visual_panels")
    return out


def training_panel(img, depth_gt, depth_pred, conf, mask):
    """img (3,H,W) float32 normalised as train_data.to_device leaves it, depth_gt / depth_pred /
    conf (H,W) float32, mask (H,W) bool or uint8, contiguous CUDA tensors on one device ->
    (H, 4W, 3) uint8 on that device."""
    shape = _map_shape("depth_gt", depth_gt)
    f32 = (torch.float32,)
    dev = depth_gt.device
    _check("depth_gt", depth_gt, f32, shape, None)
    _check("img", img, f32, (3,) + shape, dev)
    _check("depth_pred", depth_pred, f32, shape, dev)
    _check("conf", conf, f32, shape, dev)
    _check("mask", mask, (torch.bool, torch.uint8), shape, dev)
    return _panels(img, depth_gt, depth_pred, conf, mask, shape, dev)


# ToTensor's uint8 -> float32 (u / 255, divided on the host as ToTensor divides), by lookup
_TO_TENSOR = torch.arange(256, dtype=torch.uint8).float().div(255)
_TO_TENSOR_ON = {}


def _to_tensor(u8):
    """(H,W,3) uint8 -> (3,H,W) float32, ToTensor's values."""
    lut = _TO_TENSOR_ON.get(u8.device)
    if lut is None:
        lut = _TO_TENSOR_ON[u8.device] = _TO_TENSOR.to(u8.device)
    return lut[u8.long()].permute(2, 0, 1).contiguous()


def visualize_depth(depth):
    """utils/visualization.py visualize_depth on the device: (H,W) float32 CUDA tensor ->
    (3,H,W) float32, min-max normalised over the positive values, cv2 JET."""
    shape = _map_shape("depth", depth)
    _check("depth", depth, (torch.float32,), shape, None)
    return _to_tensor(_panels(None, depth, None, None, None, shape, depth.device))


def visualize_prob(prob):
    """utils/visualization.py visualize_prob on the device: (H,W) float32 CUDA tensor in 0..1 ->
    (3,H,W) float32, cv2 BONE of the grey level uint8(255 * prob)."""
    shape = _map_shape("prob", prob)
    _check("prob", prob, (torch.float32,), shape, None)
    return _to_tensor(_panels(None, None, None, prob, None, shape, prob.device))
