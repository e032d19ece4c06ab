"""CostRegNet's fused tail (conv3d_tail.cu: conv11 + prob in one kernel, u11 never stored)
against the two-layer path, bit for bit: the logits of casmvs_costreg_fwd with and without
CASMVS_FUSED_TAIL at the cascade stage shapes of 640x512 / V=3, 1152x864 / V=5 and
1920x1056 / V=7, and at ragged ones (B = 2, D = 8, h and w multiples of 8 but not of 16, several
depth chunks per tile).  The CPU part pins the coverage answer and the flag plumbing."""
import ctypes
import os
import re

import pytest
import torch

from casmvsnet_pl_b200 import ABN, _lib, ops

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHAPES = {   # (Cin, B, D, h, w)
    "640x512_stage1": (32, 1, 48, 128, 160),
    "640x512_stage2": (16, 1, 32, 256, 320),
    "640x512_stage3": (8, 1, 8, 512, 640),
    "1152x864_stage1": (32, 1, 48, 216, 288),
    "1152x864_stage2": (16, 1, 32, 432, 576),
    "1152x864_stage3": (8, 1, 8, 864, 1152),
    "1920x1056_stage1": (32, 1, 64, 264, 480),
    "1920x1056_stage2": (16, 1, 32, 528, 960),
    "1920x1056_stage3": (8, 1, 8, 1056, 1920),
    "640x512_stage1_B2": (32, 2, 48, 128, 160),
    # h % 16 == 8 (a partial last prob tile in h); w / 2 % 8 == 4 (a partial last conv11 tile)
    "ragged_h40_w56": (8, 1, 8, 40, 56),
    "ragged_B2_h24_w40": (16, 2, 16, 24, 40),
    # few tiles, D = 48: many depth chunks per tile
    "chunks_d48_h16_w24": (32, 1, 48, 16, 24),
    "tiny_d8_h8_w8": (8, 1, 8, 8, 8),
}


def _net_params(cin, seed):
    """A CostRegNet with TF32-exact weights and non-trivial folded scale / shift, so that
    negative pre-activations reach the LeakyReLU branch."""
    from casmvsnet_pl_b200.models.mvsnet import CostRegNet
    torch.manual_seed(seed)
    net = CostRegNet(cin, ABN)
    with torch.no_grad():
        for m in net.modules():
            if hasattr(m, "running_mean"):
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0.0, 0.3)
                m.running_mean.normal_(0.0, 0.3)
                m.running_var.uniform_(0.5, 1.5)
            elif isinstance(m, (torch.nn.Conv3d, torch.nn.ConvTranspose3d)):
                m.weight.copy_(_tf32(m.weight))
        net.prob.bias.normal_(0.0, 0.5)
    return net.eval().to(DEV).requires_grad_(False).packed_params()


def _tf32(t):
    """Round to nearest TF32 (ties away), as cvt.rna.tf32.f32."""
    b = t.contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
def test_fused_tail_logits_are_bit_identical(shape):
    cin, B, D, h, w = SHAPES[shape]
    assert ops.costreg_blocked_supported(cin, ops.TF32)
    assert _lib.load().casmvs_costreg_tail_supported(cin, ops.TF32) == 1
    params = _net_params(cin, cin + D + h)
    g = torch.Generator(device=DEV).manual_seed(cin * 1000 + D + w)
    x = _tf32(torch.randn(B, cin // 4, D, h, w, 4, generator=g, device=DEV))
    f0 = _lib.fallback_count()
    fused = ops.costreg(x, params, cin, ops.TF32, blocked=True, fused_tail=True)
    unfused = ops.costreg(x, params, cin, ops.TF32, blocked=True, fused_tail=False)
    torch.cuda.synchronize()
    assert _lib.fallback_count() == f0
    assert torch.isfinite(unfused).all() and unfused.std() > 0
    diff = (fused != unfused)
    assert torch.equal(fused, unfused), (
        f"{shape}: {int(diff.sum())} of {diff.numel()} logits differ, first at (b,d,h,w)="
        f"{tuple(int(i) for i in diff.nonzero()[0])}")


@pytest.mark.gpu
def test_layer_entry_point_runs_the_tail_on_the_workspace():
    """casmvs_costreg_layer_fwd(11) on the activations a two-layer call left in the workspace
    reproduces that call's logits."""
    cin, B, D, h, w = 16, 1, 16, 48, 64
    lib = _lib.load()
    params = _net_params(cin, 7)
    g = torch.Generator(device=DEV).manual_seed(7)
    x = _tf32(torch.randn(B, cin // 4, D, h, w, 4, generator=g, device=DEV))
    ws_bytes = lib.casmvs_costreg_workspace_bytes(B, cin, D, h, w)
    ws = torch.empty(ws_bytes // 4, device=DEV)
    want = torch.empty(B, D, h, w, device=DEV)
    got = torch.full_like(want, float("nan"))
    prec = ops.TF32 | ops.BLOCKED
    args = (B, cin, D, h, w, prec, ops._ptr(ws), ws_bytes)
    _lib.check(lib.casmvs_costreg_fwd(ops._ptr(x), ops._ptr(params), ops._ptr(want), *args,
                                      ops._stream()), "costreg")
    _lib.check(lib.casmvs_costreg_layer_fwd(ops._ptr(x), ops._ptr(params), ops._ptr(got), *args,
                                            11, ops._stream()), "costreg_layer")
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_tail_coverage_and_flag_are_pinned():
    """The fused tail runs exactly where the activations are blocked (TF32, Cin in {8, 16, 32});
    the flag matches the header and collides with no other precision bit."""
    lib = _lib.load()
    for cin in range(4, 65, 4):
        for prec in (_lib.FP32, _lib.TF32):
            want = int(prec == _lib.TF32 and cin in (8, 16, 32))
            assert lib.casmvs_costreg_tail_supported(cin, prec) == want, (cin, prec)
    src = open(os.path.join(ROOT, "include", "casmvs.h")).read()
    assert int(re.search(r"#define\s+CASMVS_FUSED_TAIL\s+(\d+)", src).group(1)) == _lib.FUSED_TAIL
    assert ops.FUSED_TAIL == _lib.FUSED_TAIL
    assert _lib.FUSED_TAIL & (0xff | _lib.BLOCKED | _lib.KEEP_FP32_OUT) == 0


def test_layer_entry_point_validates_before_device_work():
    from casmvsnet_pl_b200 import _lib
    lib = _lib.load()
    one = ctypes.c_void_p(16)
    rc = lib.casmvs_costreg_layer_fwd(one, one, one, 1, 8, 8, 16, 16, _lib.TF32, one, 1 << 40,
                                      12, None)
    assert rc < 0 and b"out of range" in lib.casmvs_last_error()
    rc = lib.casmvs_costreg_layer_fwd(one, one, one, 1, 8, 8, 16, 16, _lib.FP32, one, 1 << 40,
                                      11, None)
    assert rc < 0 and b"no fused" in lib.casmvs_last_error()
    rc = lib.casmvs_costreg_layer_fwd(one, one, one, 1, 12, 8, 16, 16, _lib.TF32, one, 1 << 40,
                                      11, None)
    assert rc < 0 and b"no fused" in lib.casmvs_last_error()
