"""The ring of the persistent wgmma convolution kernels across work items: a CTA runs items
blockIdx.x, blockIdx.x + gridDim.x, ... and carries its slot position and barrier parity from
one item to the next.  With CASMVS_TMA_DCHUNK=1 (one M-space depth slice per item; the fused
tail: one u9 slice) and shapes with more items than the grid has CTAs, every CTA walks several
items.  Chunking does not change the arithmetic, so each output must equal, bit for bit, the
same call with the default chunking:

  * stride 2 (conv3d_tma2.cu), channels-last and blocked;
  * transposed (conv3d_tma2.cu), channels-last and blocked;
  * 5x5 stride 2 (conv3d_tma2.cu, FeatureNet);
  * the fused conv11 + prob tail (conv3d_tail.cu).

The stride-1 kernel is covered by test_gpu_conv_fp64.py::test_stride1_several_items_per_cta."""
import os
import subprocess
import sys

import pytest
import torch

from casmvsnet_pl_b200 import ABN, ops

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLOPE = 0.01
# A CTA of the persistent kernels has 288 threads, so an SM holds at most 2048 // 288 of them:
# the grid has at most that many CTAs per SM.
MAX_CTAS_PER_SM = 2048 // 288

CONV = {   # name: kind, cin, cout, B, input (D, h, w), with a skip
    "stride2": (ops.CONV, 8, 16, 2, (32, 128, 160), False),
    "transposed": (ops.CONV_TRANSPOSE, 32, 16, 2, (16, 64, 80), True),
}
P5 = (8, 16, 3, 512, 640)   # 5x5 stride 2: cin, cout, images, h, w
WS = (8, 1, 16, 256, 320)   # CostRegNet workspace: Cin, B, D, h, w
WS_LAYERS = {"stride2_blocked": 1, "transposed_blocked": 9, "tail": 11}


def _ceil(a, b):
    return -(-a // b)


def _items(B, depth, h, w):
    """Work items at one depth slice per item, as the launchers count them: 8 x 16 tiles of the
    M space (the output of a stride-2 conv, the input of a transposed one)."""
    return B * depth * _ceil(w, 8) * _ceil(h, 16)


def _tf32(t):
    b = t.contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def _randn(g, *shape, scale=1.0):
    return _tf32(torch.randn(*shape, generator=g, device=DEV) * scale)


def _net_params(cin):
    from casmvsnet_pl_b200.models.mvsnet import CostRegNet
    torch.manual_seed(cin)
    net = CostRegNet(cin, ABN)
    with torch.no_grad():
        for m in net.modules():
            if hasattr(m, "running_mean"):
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0.0, 0.3)
                m.running_mean.normal_(0.0, 0.3)
                m.running_var.uniform_(0.5, 1.5)
    return net.eval().to(DEV).requires_grad_(False).packed_params()


def _outputs():
    """Every case's output, in the order of CONV, P5, WS_LAYERS (run in a child process)."""
    from casmvsnet_pl_b200 import _lib
    out = []
    for i, (kind, cin, cout, B, dims, skip) in enumerate(CONV.values()):
        g = torch.Generator(device=DEV).manual_seed(10 + i)
        x = _randn(g, B, *dims, cin)
        shape = (cout, cin, 3, 3, 3) if kind == ops.CONV else (cin, cout, 3, 3, 3)
        wp = ops.pack_conv3d_weight(_randn(g, *shape, scale=(27 * cin) ** -0.5), kind)
        scale = torch.rand(cout, generator=g, device=DEV) + 0.5
        shift = torch.randn(cout, generator=g, device=DEV) * 0.1
        sk = None
        if skip:
            sk = ops.as_volume_view(_randn(g, B, *(2 * d for d in dims), cout))
        y = ops.conv3d(ops.as_volume_view(x), wp, cin, cout, scale, shift, SLOPE, sk, kind, 2,
                       ops.TF32)
        out.append(ops.volume_storage(y).cpu())
    cin, cout, N, h, w = P5
    g = torch.Generator(device=DEV).manual_seed(20)
    x = _randn(g, N, h, w, cin).permute(0, 3, 1, 2)
    wp = ops.pack_conv2d_5x5s2_weight(_randn(g, cout, cin, 5, 5, scale=(25 * cin) ** -0.5))
    shift = torch.randn(cout, generator=g, device=DEV) * 0.1
    out.append(ops.conv2d_5x5s2(x, wp, shift, SLOPE, round_tf32=True).cpu())
    # blocked layers of the CostRegNet driver, on a workspace of random activations
    cin, B, D, h, w = WS
    lib = _lib.load()
    params = _net_params(cin)
    ws_bytes = lib.casmvs_costreg_workspace_bytes(B, cin, D, h, w)
    ws = _randn(torch.Generator(device=DEV).manual_seed(30), ws_bytes // 4)
    x = torch.empty(B, cin // 4, D, h, w, 4, device=DEV)
    logits = torch.full((B, D, h, w), float("nan"), device=DEV)
    for layer in WS_LAYERS.values():
        _lib.check(lib.casmvs_costreg_layer_fwd(ops._ptr(x), ops._ptr(params), ops._ptr(logits),
                                                B, cin, D, h, w, ops.TF32 | ops.BLOCKED,
                                                ops._ptr(ws), ws_bytes, layer, ops._stream()),
                   "costreg_layer")
    n = B * D * h * w
    out.append(ws[8 * n:10 * n].cpu())                         # c1 (layer 1)
    out.append(ws[ws.numel() - 64 - 8 * n:ws.numel() - 64].cpu())   # u11 (layer 9)
    out.append(logits.cpu())                                  # the tail
    torch.cuda.synchronize()
    return out


def _run(tmp_path, tag, dchunk):
    code = ("import sys, torch\n"
            "sys.path.insert(0, %r)\n"
            "sys.path.insert(0, %r)\n"
            "import test_gpu_conv_pipeline as T\n"
            "with torch.no_grad():\n"
            "    torch.save(T._outputs(), sys.argv[1])\n"
            % (ROOT, os.path.join(ROOT, "tests")))
    path = str(tmp_path / f"{tag}.pt")
    env = {k: v for k, v in os.environ.items() if k != "CASMVS_TMA_DCHUNK"}
    if dchunk:
        env["CASMVS_TMA_DCHUNK"] = str(dchunk)
    subprocess.run([sys.executable, "-c", code, path], check=True, env=env, timeout=600)
    return torch.load(path)


def test_several_items_per_cta_match_default_chunking(tmp_path):
    max_grid = torch.cuda.get_device_properties(0).multi_processor_count * MAX_CTAS_PER_SM
    items = {}
    for name, (kind, cin, cout, B, (D, h, w), _) in CONV.items():
        # the M space: the output of a stride-2 conv, the input of a transposed one
        m = (D // 2, h // 2, w // 2) if kind == ops.CONV else (D, h, w)
        items[name] = _items(B, *m)
    cin, cout, N, h, w = P5
    items["5x5s2"] = _items(1, N, _ceil(h, 2), _ceil(w, 2))
    cin, B, D, h, w = WS
    items["stride2_blocked"] = _items(B, D // 2, h // 2, w // 2)
    items["transposed_blocked"] = _items(B, D // 2, h // 2, w // 2)
    items["tail"] = _items(B, D // 2, h, w)                  # prob tiles x u9 slices
    for name, n in items.items():
        assert n > max_grid, f"{name}: {n} work items fit one round of {max_grid} CTAs"
    want = _run(tmp_path, "default", None)
    got = _run(tmp_path, "dchunk1", 1)
    assert len(got) == len(want) == len(items)
    for name, a, b in zip(items, got, want):
        assert torch.isfinite(b).all() and b.std() > 0, name
        assert torch.equal(a, b), f"{name}: {int((a != b).sum())} of {a.numel()} values differ"
