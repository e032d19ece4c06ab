"""H100-native cascade-MVS depth engine (hot path of kwea123/CasMVSNet_pl).

Public surface mirrors the reference's Python boundary (SURVEY.md §8b):
``casmvsnet_pl_b200.models.mvsnet.CascadeMVSNet`` and
``casmvsnet_pl_b200.models.modules.{homo_warp, get_depth_values, depth_regression,
ConvBnReLU, ConvBnReLU3D}``; a top-level ``models`` package re-exports them so
``from models.mvsnet import CascadeMVSNet`` (train.py:9, eval.py:11) resolves.
"""
from .norm_act import ABN, InPlaceABN  # noqa: F401

__version__ = "0.1.0"
