"""Bit-reproducible training, CPU side: the train.py flags and their defaults, the float64
weight-gradient reference against torch autograd, and the deterministic entry points' argument
checks and workspace queries (no kernel runs: there is no GPU in this tier)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from casmvsnet_pl_b200 import train
from oracle import conv3d_fp64 as K
from oracle import conv3d_wgrad_fp64 as WG

# build_parser().parse_args([]) before the two flags existed
PARENT_DEFAULTS = dict(
    root_dir="/home/ubuntu/data/mvs_training/dtu/", dataset_name="dtu", train_list=None,
    val_list=None, n_views=3, levels=3, depth_interval=2.65, n_depths=[8, 32, 48],
    interval_ratios=[1.0, 2.0, 4.0], num_groups=1, loss_type="sl1", batch_size=1, num_epochs=16,
    num_gpus=1, ckpt_path="", prefixes_to_ignore=["loss"], optimizer="sgd", lr=1e-3,
    momentum=0.9, weight_decay=1e-5, lr_scheduler="steplr", warmup_multiplier=1.0,
    warmup_epochs=0, decay_step=[20], decay_gamma=0.1, poly_exp=0.9, use_amp=False,
    exp_name="exp", precision="fp32", log_every=10, num_workers=4)


def test_flags_default_off_and_leave_other_defaults():
    a = vars(train.build_parser().parse_args([]))
    assert a.pop("deterministic") is False and a.pop("seed") is None
    assert a == PARENT_DEFAULTS


def test_flags_parse():
    a = train.build_parser().parse_args(["--deterministic", "--seed", "7"])
    assert a.deterministic is True and a.seed == 7
    with pytest.raises(SystemExit):
        train.build_parser().parse_args(["--seed", "x"])


def _torch_wgrad(kind, stride, B, cin, cout, D, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cin, D, h, w, generator=g, dtype=torch.float64)
    if kind == K.CONV:
        wt = torch.randn(cout, cin, 3, 3, 3, generator=g, dtype=torch.float64, requires_grad=True)
        y = F.conv3d(x, wt, None, stride, 1)
    else:
        wt = torch.randn(cin, cout, 3, 3, 3, generator=g, dtype=torch.float64, requires_grad=True)
        y = F.conv_transpose3d(x, wt, None, 2, 1, 1)
    gy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (y * gy).sum().backward()
    cl = lambda t: t.permute(0, 2, 3, 4, 1).contiguous()      # noqa: E731
    return cl(x), cl(gy), K.pack_weight(wt.grad, kind)


@pytest.mark.parametrize("kind,stride,B,cin,cout,D,h,w", [
    (K.CONV, 1, 2, 3, 5, 4, 6, 7), (K.CONV, 1, 1, 8, 1, 3, 5, 4), (K.CONV, 2, 2, 4, 6, 6, 8, 10),
    (K.CONV, 2, 1, 3, 2, 5, 7, 9), (K.CONV_TRANSPOSE, 2, 2, 6, 4, 3, 4, 5),
    (K.CONV_TRANSPOSE, 2, 1, 2, 3, 1, 2, 3)])
def test_wgrad_ref_matches_torch_autograd(kind, stride, B, cin, cout, D, h, w):
    x, gy, want = _torch_wgrad(kind, stride, B, cin, cout, D, h, w, seed=cin * 31 + cout)
    got = WG.wgrad_ref(x, gy, kind, stride)
    assert got.shape == (27, cin, cout)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
    A = WG.wgrad_magnitude(x, gy, kind, stride)
    assert bool((A >= got.abs() - 1e-12).all())
    ok, worst = WG.wgrad_bound_excess(got.float(), got, A, 2.0 ** -23)
    assert ok, worst
    bad = got.float().clone()
    bad[3, 0, 0] += 1e-3 * A[3, 0, 0].item() + 1e-3
    ok, worst = WG.wgrad_bound_excess(bad, got, A, 2.0 ** -20)
    assert not ok and worst["at"] == (3, 0, 0)


def test_det_entries_validate_before_any_cuda_call():
    from casmvsnet_pl_b200 import _lib
    lib = _lib.load()
    one = ctypes.c_void_p(256)
    rc = lib.casmvs_warp_cost_bwd_det(None, one, one, one, one, 1, 3, 8, 4, 8, 8, 1, one, 1 << 30, None)
    assert rc < 0 and b"null" in lib.casmvs_last_error()
    rc = lib.casmvs_warp_cost_bwd_det(one, one, one, one, one, 1, 3, 12, 4, 8, 8, 1, one, 1 << 30, None)
    assert rc < 0 and b"bad dims" in lib.casmvs_last_error()
    rc = lib.casmvs_warp_cost_bwd_det(ctypes.c_void_p(8), one, one, one, one, 1, 3, 8, 4, 8, 8, 1, one,
                                      1 << 30, None)
    assert rc < 0 and b"aligned" in lib.casmvs_last_error()
    rc = lib.casmvs_conv3d_wgrad_det(one, one, one, 1, 8, 8, 8, 8, 8, 4, 4, 4, 1, one, 1 << 30, None)
    assert rc < 0 and b"output dims" in lib.casmvs_last_error()
    rc = lib.casmvs_conv3d_wgrad_det(one, one, one, 1, 8, 8, 8, 8, 8, 8, 8, 8, 1, one, 0, None)
    assert rc < 0 and b"workspace" in lib.casmvs_last_error()
    rc = lib.casmvs_upsample2x_bilinear_bwd(one, one, 1, 8, 4, 4, 5, None)
    assert rc < 0 and b"layout" in lib.casmvs_last_error()


def test_wgrad_det_workspace_depends_on_voxel_count_only():
    from casmvsnet_pl_b200 import _lib
    lib = _lib.load()
    q = lib.casmvs_conv3d_wgrad_det_workspace_bytes
    assert q(1, 8, 8, 8, 512, 640) == q(2, 8, 8, 4, 512, 640) == q(1, 8, 8, 16, 256, 640)
    # one chunk per 64 tiles of 32 voxels, at most 2048 chunks
    assert q(1, 8, 16, 4, 256, 320) == (4 * 256 * 320 // 2048) * 27 * 8 * 16 * 4
    assert q(1, 64, 64, 1, 16, 20) == 27 * 64 * 64 * 4
    assert q(1, 8, 8, 64, 1024, 1280) == 2048 * 27 * 8 * 8 * 4
    assert q(0, 8, 8, 8, 8, 8) == 0
