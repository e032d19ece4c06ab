"""The stride-2 CostRegNet convolutions (conv1 8->16, conv3 16->32, conv5 32->64) on blocked
input: each channel quad of an input slice arrives as one contiguous run of 18 voxels x 33 rows
and is split into its even / odd column planes in shared memory, so the GEMM sees the operands
of the channels-last path (two strided loads per quad) in the same order.  Both layouts must
give the same bits.

The blocked layers run through casmvs_costreg_layer_fwd on the driver's own activations, at the
three cfg2 stage shapes and at ragged ones: tiles cut by the right and bottom edges (W not a
multiple of 16, h not a multiple of 32), odd output depths, heights and widths, a single partial
tile, B = 2.  The driver takes D, h, w in multiples of 8, so a blocked stride-2 input always has
an even depth and width."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from casmvsnet_pl_b200 import ABN, _lib, ops                 # noqa: E402
from casmvsnet_pl_b200.models.mvsnet import CostRegNet      # noqa: E402

DEV = "cuda:0"


def from_blocked(x):
    """contiguous (B,C/4,D,h,w,4) -> (B,D,h,w,C) channels-last storage."""
    B, Q, D, h, w, _ = x.shape
    return x.permute(0, 2, 3, 4, 1, 5).reshape(B, D, h, w, 4 * Q).contiguous()


def tf32(t):
    return ((t.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def _workspace_views(ws, B, D, h, w):
    """The blocked activations c0 .. c5 in casmvs_costreg_fwd's workspace (api.cu)."""
    n = B * D * h * w
    sizes = (8 * n, 2 * n, 2 * n, n // 2, n // 2, n // 8)
    shapes = ((B, 2, D, h, w, 4), (B, 4, D // 2, h // 2, w // 2, 4),
              (B, 4, D // 2, h // 2, w // 2, 4), (B, 8, D // 4, h // 4, w // 4, 4),
              (B, 8, D // 4, h // 4, w // 4, 4), (B, 16, D // 8, h // 8, w // 8, 4))
    out, off = [], 0
    for s, shp in zip(sizes, shapes):
        out.append(ws[off:off + s].view(shp))
        off += s
    return out


@pytest.mark.parametrize("B,cin,D,h,w", [
    (1, 32, 48, 128, 160),  # cfg2 stage 1 (level 2)
    (1, 16, 32, 256, 320),  # cfg2 stage 2 (level 1)
    (1, 8, 8, 512, 640),    # cfg2 stage 3 (level 0)
    (1, 8, 24, 40, 56),     # ragged last tiles; conv5 -> 3 x 5 x 7
    (2, 16, 16, 24, 40),    # B = 2; conv5 -> 2 x 3 x 5
    (2, 32, 8, 8, 8),       # conv3 and conv5 on one partial tile
])
def test_costreg_stride2_layers_blocked_equal_channels_last(B, cin, D, h, w):
    """conv1, conv3 and conv5 of the driver (blocked activations in its workspace) against the
    same layers fed the channels-last copy of their input."""
    torch.manual_seed(cin + D)
    net = CostRegNet(cin, ABN)
    with torch.no_grad():
        for m in net.modules():
            if hasattr(m, "running_mean"):
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0.0, 0.1)
    params = net.eval().to(DEV).requires_grad_(False).packed_params()
    lib = _lib.load()
    x = tf32(torch.randn(B, cin // 4, D, h, w, 4, device=DEV))
    ws_bytes = lib.casmvs_costreg_workspace_bytes(B, cin, D, h, w)
    ws = torch.empty(ws_bytes // 4, device=DEV)
    logits = torch.empty(B, D, h, w, device=DEV)
    a = (ops._ptr(x), ops._ptr(params), ops._ptr(logits), B, cin, D, h, w,
         ops.TF32 | ops.BLOCKED, ops._ptr(ws), ws_bytes)
    with torch.no_grad():
        _lib.check(lib.casmvs_costreg_fwd(*a, ops._stream()), "costreg")
        acts = _workspace_views(ws, B, D, h, w)
        for layer in (1, 3, 5):
            L = ops.costreg_layer_info(cin, layer)
            assert L["stride"] == 2 and L["kind"] == ops.CONV
            wp = params[L["w_off"]:L["w_off"] + 27 * L["cin"] * L["cout"]]
            sc = params[L["scale_off"]:L["scale_off"] + L["cout"]]
            sh = params[L["shift_off"]:L["shift_off"] + L["cout"]]
            xin = from_blocked(acts[layer - 1])
            want = ops.volume_storage(ops.conv3d(ops.as_volume_view(xin), wp, L["cin"], L["cout"],
                                                 sc, sh, 0.01, None, ops.CONV, 2, ops.TF32))
            acts[layer].fill_(float("nan"))
            _lib.check(lib.casmvs_costreg_layer_fwd(*a, layer, ops._stream()), "costreg_layer")
            torch.cuda.synchronize()
            assert torch.equal(from_blocked(acts[layer]), want), f"layer {layer}"
