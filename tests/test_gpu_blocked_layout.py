"""The blocked activation layout of the TF32 CostRegNet path, (B, C/4, D, h, w, 4): the same
kernels and arithmetic as the channels-last layout, only the addresses differ, so the results
must be bit-identical to the channels-last per-layer path."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from casmvsnet_pl_b200 import ABN, _lib, ops, synth          # noqa: E402
from casmvsnet_pl_b200.models.mvsnet import CostRegNet      # noqa: E402

DEV = "cuda:0"


def to_blocked(x_ndhwc):
    """(B,D,h,w,C) channels-last storage -> contiguous (B,C/4,D,h,w,4)."""
    B, D, h, w, C = x_ndhwc.shape
    return x_ndhwc.reshape(B, D, h, w, C // 4, 4).permute(0, 4, 1, 2, 3, 5).contiguous()


def test_blocked_flag_matches_header():
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "include", "casmvs.h")).read()
    assert int(re.search(r"#define\s+CASMVS_BLOCKED\s+(\d+)", src).group(1)) == _lib.BLOCKED
    # OR-ed into a precision / a rounding flag: must not collide with them
    assert _lib.BLOCKED & (0xff | _lib.ROUND_TF32 | _lib.KEEP_FP32_OUT) == 0


def _costreg_chain(x_ndhwc, params, cin):
    """The 11 layers one at a time through the public (channels-last) conv entry point, in the
    order and with the skips of casmvs_costreg_fwd."""
    info = [ops.costreg_layer_info(cin, i) for i in range(11)]

    def layer(i, x, skip=None, slope=0.01):
        L = info[i]
        w = params[L["w_off"]:L["w_off"] + 27 * L["cin"] * L["cout"]]
        sc = params[L["scale_off"]:L["scale_off"] + L["cout"]]
        sh = params[L["shift_off"]:L["shift_off"] + L["cout"]]
        return ops.conv3d(x, w, L["cin"], L["cout"], sc, sh, slope, skip, L["kind"], L["stride"],
                          ops.TF32)

    c0 = layer(0, ops.as_volume_view(x_ndhwc))
    c2 = layer(2, layer(1, c0))
    c4 = layer(4, layer(3, c2))
    c6 = layer(6, layer(5, c4))
    u = layer(7, c6, c4)
    u = layer(8, u, c2)
    u = layer(9, u, c0)
    return layer(10, u, slope=1.0).squeeze(1)


def _net(cin):
    torch.manual_seed(cin)
    net = CostRegNet(cin, ABN)
    with torch.no_grad():                 # non-trivial folded scale / shift in every epilogue
        for m in net.modules():
            if hasattr(m, "running_mean"):
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0.0, 0.1)
                m.running_mean.normal_(0.0, 0.1)
                m.running_var.uniform_(0.5, 1.5)
    net = net.eval().to(DEV).requires_grad_(False)
    net.precision = "tf32"
    return net


@pytest.mark.parametrize("cin,B", [(8, 1), (16, 1), (32, 1), (8, 2), (32, 2)])
def test_costreg_blocked_equals_channels_last_chain(cin, B):
    net = _net(cin)
    assert net.blocked_supported()
    D, h, w = 16, 40, 56                  # 40 x 56: tiles cut by the image edge at every level
    x = torch.randn(B, D, h, w, cin, device=DEV)
    params = net.packed_params()
    with torch.no_grad():
        want = _costreg_chain(x, params, cin)
        got_blocked = net.forward_blocked(to_blocked(x))
        got_cl = net(ops.as_volume_view(x)).squeeze(1)      # channels-last input, blocked inside
    torch.cuda.synchronize()
    assert got_blocked.shape == want.shape == (B, D, h, w)
    assert torch.equal(got_blocked, want)
    assert torch.equal(got_cl, want)


@pytest.mark.parametrize("cin", [4, 12])
def test_costreg_uncovered_conv0_stays_channels_last(cin):
    """A conv0 input width no tensor-core kernel covers (e.g. 4 group-wise correlation groups):
    the driver keeps every activation channels-last, conv0 runs on the CUDA cores (counted),
    and the result is the per-layer chain's."""
    net = _net(cin)
    assert not net.blocked_supported()
    x = torch.randn(1, 16, 40, 56, cin, device=DEV)
    params = net.packed_params()
    with torch.no_grad():
        want = _costreg_chain(x, params, cin)
        f0 = _lib.fallback_count()
        got = net(ops.as_volume_view(x)).squeeze(1)
        torch.cuda.synchronize()
        assert _lib.fallback_count() - f0 == 1                 # conv0 only
        with pytest.raises(_lib.CasMVSError):
            net.forward_blocked(torch.zeros(1, cin // 4, 16, 40, 56, 4, device=DEV))
    assert torch.equal(got, want)


def test_costreg_blocked_input_is_validated():
    net = _net(8)
    with pytest.raises(ValueError):
        net.forward_blocked(torch.zeros(1, 8, 8, 8, 8, device=DEV))   # channels-last shape
    net.precision = "fp32"
    with pytest.raises(_lib.CasMVSError):
        net.forward_blocked(torch.zeros(1, 2, 8, 8, 8, 4, device=DEV))


@pytest.mark.parametrize("V,C,G,B", [(3, 8, 1, 1), (3, 16, 1, 1), (3, 32, 1, 1), (2, 16, 1, 1),
                                     (3, 8, 8, 1), (3, 16, 8, 1), (3, 32, 8, 1), (2, 32, 8, 1),
                                     (3, 16, 1, 2), (3, 32, 8, 2)])
def test_warp_cost_ladder_blocked_equals_channels_last(V, C, G, B):
    level = {8: 0, 16: 1, 32: 2}[C]
    g = torch.Generator().manual_seed(7 + C + G)
    h, w = (512 >> level) - 3, (640 >> level) - 5       # ragged tiles at the right/bottom edge
    D = {0: 8, 1: 16, 2: 24}[level]
    feats = torch.randn(B, V, C, h, w, generator=g)
    feats = feats.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3).to(DEV)
    pm = synth.projection_matrices(V, 640, 512)[:, level].unsqueeze(0).repeat(B, 1, 1, 1).to(DEV)
    lad = ops.Ladder(600.0, 2.65 * 2 ** level, D, B, h, w, DEV)
    with torch.no_grad():
        cl = ops.warp_cost_ladder(feats, pm, lad, G, round_tf32=True)
        blk = ops.warp_cost_ladder(feats, pm, lad, G, round_tf32=True, blocked=True)
    torch.cuda.synchronize()
    cout = C if G == 1 else G
    assert blk.shape == (B, cout // 4, D, h, w, 4)
    assert torch.equal(blk, to_blocked(ops.volume_storage(cl)))
