"""Operator surface of the reference's ``models/modules.py`` on the H100 engine.

Same names, argument meaning and shapes as the reference (SURVEY.md §8b); the
bodies call the hand-written CUDA kernels through the C ABI (../ops.py).
"""
import torch
from torch import nn

from .. import ops
from ..norm_act import ABN, InPlaceABN, activation_slope, folded_scale_shift  # noqa: F401

__all__ = ["ConvBnReLU", "ConvBnReLU3D", "get_depth_values", "homo_warp",
           "depth_regression", "InPlaceABN", "ABN"]


class ConvBnReLU(nn.Module):
    """2D conv + norm-act (reference models/modules.py:8-18).  Used only by the
    FeatureNet, which stays PyTorch/cuDNN by design (north_star: host glue)."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, pad=1,
                 norm_act=InPlaceABN):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride=stride,
                              padding=pad, bias=False)
        self.bn = norm_act(out_channels)

    def forward(self, x):
        return self.bn(self.conv(x))


class ConvBnReLU3D(nn.Module):
    """3x3x3 conv + norm-act (reference models/modules.py:21-31) as ONE fused
    CUDA kernel: conv -> x*alpha+beta -> LeakyReLU.  ``conv``/``bn`` are kept as
    parameter holders so state-dict keys match the reference's."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, pad=1,
                 norm_act=InPlaceABN):
        super().__init__()
        if kernel_size != 3 or pad != 1 or stride not in (1, 2):
            raise ValueError("the engine implements the reference's 3x3x3, pad 1, stride 1|2 conv")
        self.conv = nn.Conv3d(in_channels, out_channels, kernel_size, stride=stride,
                              padding=pad, bias=False)
        self.bn = norm_act(out_channels)
        self.precision = "fp32"
        self._packed = None
        self._packed_key = None

    def _params(self):
        key = tuple((t.data_ptr(), t._version) for t in
                    (self.conv.weight, self.bn.weight, self.bn.bias,
                     self.bn.running_mean, self.bn.running_var))
        if key != self._packed_key:
            w = ops.pack_conv3d_weight(self.conv.weight, ops.CONV)
            a, b = folded_scale_shift(self.bn)
            self._packed = (w, a, b)
            self._packed_key = key
        return self._packed

    def forward(self, x):
        if torch.is_grad_enabled() and (x.requires_grad or
                                        any(p.requires_grad for p in self.parameters())):
            from .. import autograd as AG
            return self.bn(AG.conv3d(x, self.conv.weight, ops.CONV, self.conv.stride[0],
                                     ops.PRECISIONS[self.precision]))
        if self.bn.training:
            raise ops._lib.CasMVSError("ConvBnReLU3D inference path needs .eval() (training runs "
                                       "through the autograd path: enable grad)")
        w, a, b = self._params()
        return ops.conv3d(x, w, self.conv.in_channels, self.conv.out_channels, a, b,
                          activation_slope(self.bn), None, ops.CONV, self.conv.stride[0],
                          ops.PRECISIONS[self.precision])


def get_depth_values(current_depth, n_depths, depth_interval):
    """current_depth (B,1,H,W); depth_interval (B,1) or float -> (B,D,H,W)
    (reference models/modules.py:34-49)."""
    return ops.depth_hypotheses(current_depth, n_depths, depth_interval, upsample=False)


def homo_warp(src_feat, proj_mat, depth_values):
    """src_feat (B,C,H,W), proj_mat (B,3,4), depth_values (B,D,H,W) -> (B,C,D,H,W)
    (reference models/modules.py:52-92)."""
    return ops.homo_warp(src_feat, proj_mat, depth_values)


def depth_regression(p, depth_values):
    """p (B,D,H,W) probabilities, depth_values (B,D,H,W) or (D) -> (B,H,W)
    (reference models/modules.py:95-104)."""
    depth, _, _, _ = ops.regress(p, depth_values, input_is_prob=True)
    return depth.to(depth_values.dtype)
