"""Seeded inputs of the reference cross-checks (tests/test_oracle_vs_reference.py); the
reference's outputs for them are recorded by oracle/make_golden_live.py."""
import torch

from casmvsnet_pl_b200 import synth


def predict_depth_inputs():
    g = torch.Generator().manual_seed(9)
    feats = torch.randn(2, 4, 16, 16, 24, generator=g)
    pms = synth.projection_matrices(4, W=96, H=64, stress=True, behind_view=3)[:, 1]
    pms = pms.unsqueeze(0).expand(2, -1, -1, -1).contiguous()
    dv = 430.0 + 5.3 * torch.arange(16).float().reshape(1, 16, 1, 1) + torch.rand(2, 16, 16, 24, generator=g)
    return feats, pms, dv


def feature_input():
    return torch.randn(1, 3, 32, 48, generator=torch.Generator().manual_seed(4))
