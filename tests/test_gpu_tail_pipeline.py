"""The fused conv11 + prob tail (conv3d_tail.cu) against the unfused pair, bit for bit, under
every depth chunking: prob's logit stores are deferred past the next slice's wgmma and carried
into the CTA's next work item, the wgmma of the u9 / u11 slices that lie wholly in the depth
padding at d0 = 0 are skipped, and prob's three live kd columns run as one m64n8k8.  The logits
of casmvs_costreg_layer_fwd(11) on the workspace of a two-layer call must equal that call's
logits (conv11 -> u11 -> prob) as int32,
so a signed zero or a last bit out of place fails.

Shapes: the three 640x512 stages, its full-resolution stage with B = 4 (several items per CTA,
the pending epilogue crossing items and batch entries), the full-resolution stages of 1152x864
and 1920x1056, and ragged h, w (multiples of 8, not of 16) at D = 8 and 16.  Chunkings: the
default and CASMVS_TMA_DCHUNK = 1 (every item starts or ends at the volume edge), 2, 3 (odd step
counts) and 8, each in a child process since switches are read once per process."""
import os
import subprocess
import sys

import pytest
import torch

from casmvsnet_pl_b200 import ABN, _lib, ops

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHAPES = {   # (Cin, B, D, h, w)
    "640x512_stage1": (32, 1, 48, 128, 160),
    "640x512_stage2": (16, 1, 32, 256, 320),
    "640x512_stage3": (8, 1, 8, 512, 640),
    "640x512_stage3_B4": (8, 4, 8, 512, 640),
    "1152x864_stage3": (8, 1, 8, 864, 1152),
    "1920x1056_stage3": (8, 1, 8, 1056, 1920),
    "ragged_d8_h40_w56": (8, 1, 8, 40, 56),
    "ragged_d16_B2_h24_w40": (16, 2, 16, 24, 40),
}


def _tf32(t):
    b = t.contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def _net_params(cin, seed):
    """TF32-exact weights and non-trivial folded scale / shift (both LeakyReLU branches)."""
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


def _mismatches():
    """{shape: (differing logits, total, unfused std)} under this process's chunking."""
    lib = _lib.load()
    res = {}
    for name, (cin, B, D, h, w) in SHAPES.items():
        params = _net_params(cin, cin + D + h + B)
        g = torch.Generator(device=DEV).manual_seed(cin * 1000 + D + w + B)
        x = _tf32(torch.randn(B, cin // 4, D, h, w, 4, generator=g, device=DEV))
        ws_bytes = lib.casmvs_costreg_workspace_bytes(B, cin, D, h, w)
        ws = torch.empty(ws_bytes // 4, device=DEV)
        want = torch.empty(B, D, h, w, device=DEV)
        got = torch.full_like(want, float("nan"))
        args = (B, cin, D, h, w, ops.TF32 | ops.BLOCKED, ops._ptr(ws), ws_bytes)
        f0 = _lib.fallback_count()
        _lib.check(lib.casmvs_costreg_fwd(ops._ptr(x), ops._ptr(params), ops._ptr(want), *args,
                                          ops._stream()), "costreg")
        _lib.check(lib.casmvs_costreg_layer_fwd(ops._ptr(x), ops._ptr(params), ops._ptr(got),
                                                *args, 11, ops._stream()), "costreg_layer")
        torch.cuda.synchronize()
        assert _lib.fallback_count() == f0
        diff = int((got.view(torch.int32) != want.view(torch.int32)).sum())
        res[name] = (diff, want.numel(), float(want.std()), bool(torch.isfinite(want).all()))
        del ws, x, want, got
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("dchunk", [0, 1, 2, 3, 8])
def test_fused_tail_matches_unfused_bits_under_every_chunking(tmp_path, dchunk):
    code = ("import sys, torch\n"
            "sys.path.insert(0, %r)\n"
            "sys.path.insert(0, %r)\n"
            "import test_gpu_tail_pipeline as T\n"
            "with torch.no_grad():\n"
            "    torch.save(T._mismatches(), sys.argv[1])\n"
            % (ROOT, os.path.join(ROOT, "tests")))
    path = str(tmp_path / f"dchunk{dchunk}.pt")
    env = {k: v for k, v in os.environ.items() if k != "CASMVS_TMA_DCHUNK"}
    if dchunk:
        env["CASMVS_TMA_DCHUNK"] = str(dchunk)
    subprocess.run([sys.executable, "-c", code, path], check=True, env=env, timeout=900)
    res = torch.load(path)
    assert set(res) == set(SHAPES)
    for name, (diff, n, std, finite) in res.items():
        assert finite and std > 0, name
    bad = {name: f"{diff} of {n}" for name, (diff, n, _, _) in res.items() if diff}
    assert not bad, f"CASMVS_TMA_DCHUNK={dchunk or 'default'}: logits differ: {bad}"
