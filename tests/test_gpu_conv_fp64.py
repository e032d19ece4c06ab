"""Every K2 convolution kernel element by element against the float64 reference
(oracle/conv3d_fp64.py), at the shapes the benchmark runs and at ragged ones:

  * inside the CostRegNet driver (blocked activations, caller-owned workspace): each layer
    against that layer applied in float64 to the kernel's own input activation and skip, so
    errors do not compound -- at the three cascade stages of 640x512 / V=3 and 1152x864 / V=5,
    B=2, the real blocked cost-volume producer, and the fp32 (CUDA-core, channels-last) mode;
  * through the public ops.conv3d: every layer kind in TF32, TF32 | KEEP_FP32_OUT and FP32,
    with and without skip, at the production layer shapes and at ragged ones;
  * several work items per CTA forced at a small shape (CASMVS_TMA_DCHUNK=1);
  * the FeatureNet wgmma convolutions (planar 3x3, 5x5 stride 2) at both image pyramids;
  * the backward: casmvs_conv3d_wgrad and the data gradients of autograd.Conv3dFn at a
    640x512 training crop.

Bound per element: |y - y64| <= eps * A + r * |y64| + tiny, A = |scale| * conv(|x|, |w|)
(R.bound_excess).  Inputs of the TF32 runs are TF32-exact (pre-rounded, or the previous
layer's rounded output), so the products are exact and eps measures the accumulation alone.
EPS holds, per kernel, at most 4x the worst err/A measured on an H100 over this file, and never
more than the ceilings."""
import os
import zlib

import pytest
import torch

from casmvsnet_pl_b200 import ABN, _lib, ops
from casmvsnet_pl_b200 import autograd as AG
from oracle import conv3d_fp64 as R

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

EPS_CEIL_WGMMA = 2.0 ** -14      # wgmma kernels (TF32 operands, fp32 accumulators)
EPS_CEIL_FP32 = 2.0 ** -17       # fp32 CUDA-core kernels
# Worst err/A over every case of this file (it prints them), measured on an H100 80GB HBM3 at a
# 400 W power limit; each eps is the largest power of two within 4x of it.
EPS = {
    "tma": 2.0 ** -19,           # stride-1 and planar wgmma kernel (conv3d_tma.cu): 7.3e-7
    "tma2": 2.0 ** -19,          # stride-2, transposed, 5x5 stride-2 wgmma (conv3d_tma2.cu): 5.6e-7
    "direct": 2.0 ** -20,        # fp32 CUDA-core kernel (conv3d_direct.cu): 4.5e-7
    "wgrad": 2.0 ** -19,         # weight gradient (backward.cu), per sum |x| |gy|: 8.6e-7
}

SLOPE = 0.01


def _check(tag, kernel, y, y64, A, r, extra=None):
    """Asserts the bound of R.bound_excess at EPS[kernel]; returns the eps the layer needed."""
    ok, worst = R.bound_excess(y, y64, A, EPS[kernel], r, extra)
    print(f"[fp64] {tag} [{kernel}]: worst err/A {worst['eps_needed']:.3e} "
          f"(eps {EPS[kernel]:.3e}) at (b,d,h,w,c)={worst['at']}")
    assert ok, (f"{tag} [{kernel}]: |y - y64| exceeds eps*A + r|y64| + tiny; worst voxel "
                f"(b,d,h,w,c)={worst['at']} h%16={worst['h16']} w%8={worst['w8']} "
                f"slice={worst['slice']}: got {worst['got']!r}, float64 {worst['want']!r}, "
                f"A={worst['A']:.4e}, needs eps {worst['eps_needed']:.3e} > {EPS[kernel]:.3e}")
    return worst["eps_needed"]


def _seed(*parts):
    return zlib.crc32("/".join(parts).encode())


def _is_tf32(t):
    return bool((t.contiguous().view(torch.int32) & 0x1FFF).eq(0).all())


def _randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device=DEV) * scale


# ------------------------------------------------------------------------------- hardware RNA
def test_tf32_rna_matches_the_hardware_conversion():
    """R.tf32_rna against cvt.rna.tf32.f32 itself (the rounding store of bias_lrelu_, bias 0,
    slope 1): ties, negatives, subnormals, the largest finite values, and random bits."""
    pats = [0x3F800FFF, 0x3F801000, 0x3F803000, 0x3F801001, 0xBF801000, 0xBF800FFF, 0x3FFFF000,
            0x00000FFF, 0x00001000, 0x807FF000, 0x7F7FE000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000,
            0x00000000, 0x00000001, 0x00800000, 0x4B7FF000]
    g = torch.Generator().manual_seed(0)
    rnd = torch.randint(-2 ** 31, 2 ** 31, (4096 - len(pats),), generator=g, dtype=torch.int64)
    bits = torch.cat([torch.tensor(pats, dtype=torch.int64), rnd]).to(torch.int32)
    x = bits.view(torch.float32)
    x = torch.where(torch.isnan(x), torch.zeros_like(x), x)
    dev = x.reshape(1, 4, 32, 32).to(DEV).contiguous(memory_format=torch.channels_last)
    ops.bias_lrelu_(dev, torch.zeros(4, device=DEV), 1.0, round_tf32=True)
    got = dev.permute(0, 2, 3, 1).reshape(-1).cpu()
    want = R.tf32_rna(x.reshape(1, 4, 32, 32).permute(0, 2, 3, 1).reshape(-1).contiguous())
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


# ------------------------------------------------------------------------------- ops.conv3d
LAYERS = {   # name: kind, stride, cin, cout, production input dims (cfg2: 640x512, D=48/32/8)
    "conv0_c8": (ops.CONV, 1, 8, 8, (8, 512, 640)),
    "conv0_c16": (ops.CONV, 1, 16, 8, (32, 256, 320)),
    "conv0_c32": (ops.CONV, 1, 32, 8, (48, 128, 160)),
    "conv2": (ops.CONV, 1, 16, 16, (24, 64, 80)),
    "conv4": (ops.CONV, 1, 32, 32, (12, 32, 40)),
    "conv6": (ops.CONV, 1, 64, 64, (6, 16, 20)),
    "prob": (ops.CONV, 1, 8, 1, (32, 256, 320)),
    "conv1": (ops.CONV, 2, 8, 16, (48, 128, 160)),
    "conv3": (ops.CONV, 2, 16, 32, (24, 64, 80)),
    "conv5": (ops.CONV, 2, 32, 64, (12, 32, 40)),
    "conv7": (ops.CONV_TRANSPOSE, 2, 64, 32, (6, 16, 20)),
    "conv9": (ops.CONV_TRANSPOSE, 2, 32, 16, (12, 32, 40)),
    "conv11": (ops.CONV_TRANSPOSE, 2, 16, 8, (24, 64, 80)),
}
RAGGED = {   # w % 8 != 0 and h % 16 != 0; odd D / h / w for stride 2
    (ops.CONV, 1): (5, 37, 29),
    (ops.CONV, 2): (7, 33, 27),
    (ops.CONV_TRANSPOSE, 2): (3, 19, 13),
}


def _layer_inputs(g, kind, cin, cout, dims, B=2):
    x = R.tf32_rna(_randn(g, B, *dims, cin))
    shape = (cout, cin, 3, 3, 3) if kind == ops.CONV else (cin, cout, 3, 3, 3)
    wt = R.tf32_rna(_randn(g, *shape, scale=(27 * cin) ** -0.5))
    scale = torch.rand(cout, generator=g, device=DEV) + 0.5
    shift = _randn(g, cout, scale=0.1)
    return x, wt, scale, shift


@pytest.mark.parametrize("group", ["production", "ragged"])
@pytest.mark.parametrize("name", list(LAYERS))
def test_conv3d_layer_vs_fp64(name, group):
    kind, stride, cin, cout, dims = LAYERS[name]
    if group == "ragged":
        dims = RAGGED[(kind, stride)]
    g = torch.Generator(device=DEV).manual_seed(_seed(name, group))
    x, wt, scale, shift = _layer_inputs(g, kind, cin, cout, dims)
    wp = ops.pack_conv3d_weight(wt, kind)
    w64 = R.pack_weight(wt, kind)
    acc = R.conv3d_ref(x, w64, kind, stride)
    A = R.magnitude(x, w64, kind, stride, scale)
    skip = _randn(g, *acc.shape)
    tag = f"ops.conv3d {name} {group} {tuple(x.shape)}"
    for precision in (ops.TF32, ops.TF32 | ops.KEEP_FP32_OUT, ops.FP32):
        for sk in (None, skip):
            if sk is not None and cout % 2:
                continue                      # the prob head never takes a skip
            tf32 = (precision & 0xff) == ops.TF32
            keep = bool(precision & ops.KEEP_FP32_OUT)
            # stride 2 with a skip (never used by CostRegNet) has no wgmma kernel: it runs on
            # the CUDA cores, counted as a fallback
            fallback = tf32 and kind == ops.CONV and stride == 2 and sk is not None
            kernel = "direct" if not tf32 or fallback else "tma" if stride == 1 else "tma2"
            f0 = _lib.fallback_count()
            y = ops.conv3d(ops.as_volume_view(x), wp, cin, cout, scale, shift, SLOPE,
                           None if sk is None else ops.as_volume_view(sk), kind, stride, precision)
            y = ops.volume_storage(y)
            torch.cuda.synchronize()
            assert _lib.fallback_count() - f0 == (1 if fallback else 0)
            rounded = tf32 and not keep and cout > 1
            if rounded:
                assert _is_tf32(y)
            elif tf32 and keep:
                # the fp32 accumulator is stored as is: a rounded store would pass eps*A + r|y|
                # only by chance, so say it outright
                assert not _is_tf32(y), f"{tag}: KEEP_FP32_OUT output is TF32-rounded"
            y64 = R.epilogue(acc, scale, shift, SLOPE, sk)
            _check(f"{tag} prec={precision} skip={sk is not None}", kernel, y, y64, A,
                   R.R_TF32 if rounded else 0.0, R.epilogue_magnitude(y64, shift, sk))


# ------------------------------------------------------------------------------- several items
def _dchunk_case_inputs():
    out = []
    for i, (cin, cout, dims) in enumerate([(16, 16, (24, 40, 24)), (64, 64, (12, 32, 40)),
                                           (32, 8, (20, 48, 40))]):
        g = torch.Generator(device=DEV).manual_seed(100 + i)
        x, wt, scale, shift = _layer_inputs(g, ops.CONV, cin, cout, dims)
        skip = _randn(g, 2, *dims, cout)
        out.append((cin, cout, x, wt, scale, shift, skip))
    return out


def _dchunk_case_outputs():
    """Run in a child process with CASMVS_TMA_DCHUNK=1: one output slice per work item, so
    every CTA runs several items (accumulator carry-over, deferred epilogue across items, ring
    phases) at shapes whose default chunking fits one round."""
    res = []
    for cin, cout, x, wt, scale, shift, skip in _dchunk_case_inputs():
        wp = ops.pack_conv3d_weight(wt, ops.CONV)
        y = ops.conv3d(ops.as_volume_view(x), wp, cin, cout, scale, shift, SLOPE,
                       ops.as_volume_view(skip), ops.CONV, 1, ops.TF32)
        res.append(ops.volume_storage(y).cpu())
    return res


def test_stride1_several_items_per_cta(tmp_path):
    import subprocess
    import sys
    code = ("import sys, torch\n"
            "sys.path.insert(0, %r)\n"
            "sys.path.insert(0, %r)\n"
            "import test_gpu_conv_fp64 as T\n"
            "with torch.no_grad():\n"
            "    torch.save(T._dchunk_case_outputs(), sys.argv[1])\n"
            % (ROOT, os.path.join(ROOT, "tests")))
    path = str(tmp_path / "dchunk1.pt")
    env = dict(os.environ, CASMVS_TMA_DCHUNK="1")
    subprocess.run([sys.executable, "-c", code, path], check=True, env=env, timeout=600)
    got = torch.load(path)
    for y, (cin, cout, x, wt, scale, shift, skip) in zip(got, _dchunk_case_inputs()):
        w64 = R.pack_weight(wt, ops.CONV)
        y64 = R.epilogue(R.conv3d_ref(x, w64, ops.CONV), scale, shift, SLOPE, skip)
        A = R.magnitude(x, w64, ops.CONV, 1, scale)
        _check(f"dchunk=1 conv {cin}->{cout} {tuple(x.shape)}", "tma", y.to(DEV), y64, A,
               R.R_TF32, R.epilogue_magnitude(y64, shift, skip))


# ------------------------------------------------------------------------------- CostRegNet driver
def _net_params(cin):
    from casmvsnet_pl_b200.models.mvsnet import CostRegNet
    torch.manual_seed(cin)
    net = CostRegNet(cin, ABN)
    with torch.no_grad():                 # non-trivial folded scale / shift in every epilogue
        for m in net.modules():
            if hasattr(m, "running_mean"):
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0.0, 0.1)
                m.running_mean.normal_(0.0, 0.1)
                m.running_var.uniform_(0.5, 1.5)
    return net.eval().to(DEV).requires_grad_(False).packed_params()


# activations of casmvs_costreg_fwd in workspace order: (channels, resolution divisor)
_ACTS = [("c0", 8, 1), ("c1", 16, 2), ("c2", 16, 2), ("c3", 32, 4), ("c4", 32, 4),
         ("c5", 64, 8), ("c6", 64, 8), ("u7", 32, 4), ("u9", 16, 2), ("u11", 8, 1)]
_IN = ["x", "c0", "c1", "c2", "c3", "c4", "c5", "c6", "u7", "u9", "u11"]
_OUT = ["c0", "c1", "c2", "c3", "c4", "c5", "c6", "u7", "u9", "u11", "logits"]
_SKIP = {7: "c4", 8: "c2", 9: "c0"}


def _costreg_layers_vs_fp64(tag, x, cin, B, D, h, w, precision, blocked_in):
    """Run casmvs_costreg_fwd with a caller-owned workspace, then check every layer against
    the float64 layer applied to the kernel's own input activation (and skip)."""
    lib = _lib.load()
    params = _net_params(cin)
    ws_bytes = lib.casmvs_costreg_workspace_bytes(B, cin, D, h, w)
    ws = torch.full((ws_bytes // 4,), float("nan"), device=DEV)
    logits = torch.empty(B, D, h, w, device=DEV)
    blocked = precision == ops.TF32 and ops.costreg_blocked_supported(cin, ops.TF32)
    assert blocked or not blocked_in
    f0 = _lib.fallback_count()
    _lib.check(lib.casmvs_costreg_fwd(ops._ptr(x), ops._ptr(params), ops._ptr(logits), B, cin, D,
                                      h, w, precision | (ops.BLOCKED if blocked_in else 0),
                                      ops._ptr(ws), ws_bytes, ops._stream()), "costreg")
    torch.cuda.synchronize()
    assert _lib.fallback_count() == f0
    # the activations at the offsets casmvs_costreg_fwd slices the workspace at
    n = B * D * h * w
    acts, off = {}, 0
    for name, c, s in _ACTS:
        size = c * n // s ** 3
        buf = ws[off:off + size]
        dims = (D // s, h // s, w // s)
        acts[name] = (R.from_blocked(buf.view(B, c // 4, *dims, 4)) if blocked
                      else buf.view(B, *dims, c))
        off += size
    assert (off + 64) * 4 == ws_bytes          # every float but the 64-float alignment slack
    acts["x"] = R.from_blocked(x) if blocked_in else x
    acts["logits"] = logits.unsqueeze(-1)
    tf32 = precision == ops.TF32
    for i in range(11):
        L = ops.costreg_layer_info(cin, i)
        w_ = params[L["w_off"]:L["w_off"] + 27 * L["cin"] * L["cout"]].view(27, L["cin"], L["cout"])
        scale = params[L["scale_off"]:L["scale_off"] + L["cout"]]
        shift = params[L["shift_off"]:L["shift_off"] + L["cout"]]
        xin = acts[_IN[i]]
        if tf32:
            w_ = R.tf32_rna(w_)                # the operand images hold the weights RNA-rounded
            assert _is_tf32(xin), f"{tag}: input of layer {i} is not TF32-exact"
        skip = acts[_SKIP[i]] if i in _SKIP else None
        slope = 1.0 if i == 10 else SLOPE
        acc = R.conv3d_ref(xin, w_, L["kind"], L["stride"])
        y64 = R.epilogue(acc, scale, shift, slope, skip)
        del acc
        A = R.magnitude(xin, w_, L["kind"], L["stride"], scale)
        kernel = "direct" if not tf32 else "tma" if L["stride"] == 1 else "tma2"
        rounded = tf32 and L["cout"] > 1
        _check(f"{tag} layer {i} ({_OUT[i]})", kernel, acts[_OUT[i]], y64, A,
               R.R_TF32 if rounded else 0.0, R.epilogue_magnitude(y64, shift, skip))
        del y64, A


COSTREG_SHAPES = {   # cascade stage shapes: (Cin, B, D, h, w)
    "640x512_stage1": (32, 1, 48, 128, 160),
    "640x512_stage2": (16, 1, 32, 256, 320),
    "640x512_stage3": (8, 1, 8, 512, 640),
    "640x512_gwc8_stage1": (8, 1, 48, 128, 160),
    "1152x864_stage1": (32, 1, 48, 216, 288),
    "1152x864_stage2": (16, 1, 32, 432, 576),
    "1152x864_stage3": (8, 1, 8, 864, 1152),
    "640x512_stage1_B2": (32, 2, 48, 128, 160),
}


@pytest.mark.parametrize("shape", list(COSTREG_SHAPES))
def test_costreg_driver_layers_vs_fp64(shape):
    cin, B, D, h, w = COSTREG_SHAPES[shape]
    g = torch.Generator(device=DEV).manual_seed(cin * 1000 + D)
    cost = R.tf32_rna(_randn(g, B, D, h, w, cin))          # the TF32-rounded cost volume
    _costreg_layers_vs_fp64(f"costreg tf32 {shape}", R.to_blocked(cost), cin, B, D, h, w,
                            ops.TF32, True)


def test_costreg_driver_layers_vs_fp64_from_the_cost_volume_producer():
    """The input is the blocked, TF32-rounded cost volume of warp_cost_ladder (640x512, V=3,
    coarsest stage)."""
    from casmvsnet_pl_b200 import synth
    B, V, C, D, level = 1, 3, 32, 48, 2
    h, w = 512 >> level, 640 >> level
    g = torch.Generator().manual_seed(11)
    feats = torch.randn(B, V, C, h, w, generator=g)
    feats = feats.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3).to(DEV)
    pm = synth.projection_matrices(V, 640, 512)[:, level].unsqueeze(0).to(DEV)
    lad = ops.Ladder(600.0, 2.65 * 2 ** level, D, B, h, w, DEV)
    cost = ops.warp_cost_ladder(feats, pm, lad, 1, round_tf32=True, blocked=True)
    _costreg_layers_vs_fp64("costreg tf32 warp_cost_ladder 640x512 stage1", cost, C, B, D, h, w,
                            ops.TF32, True)


@pytest.mark.parametrize("shape", ["640x512_stage1", "640x512_stage3"])
def test_costreg_driver_layers_vs_fp64_fp32_mode(shape):
    cin, B, D, h, w = COSTREG_SHAPES[shape]
    g = torch.Generator(device=DEV).manual_seed(cin * 1000 + D + 1)
    cost = _randn(g, B, D, h, w, cin)
    _costreg_layers_vs_fp64(f"costreg fp32 {shape}", cost, cin, B, D, h, w, ops.FP32, False)


# ------------------------------------------------------------------------------- FeatureNet
PYRAMIDS = {"640x512_V3": (3, 512, 640), "1152x864_V5": (5, 864, 1152)}
# (cin, cout, resolution divisor): conv0.1, conv1.1/1.2, conv2.1/2.2, smooth1, smooth0
PLANAR = [(8, 8, 1), (16, 16, 2), (32, 32, 4), (32, 16, 2), (32, 8, 1)]
P5 = [(8, 16, 1), (16, 32, 2)]          # conv1.0, conv2.0: input resolution divisor


@pytest.mark.parametrize("pyramid", list(PYRAMIDS))
def test_featurenet_wgmma_convs_vs_fp64(pyramid):
    N, H, W = PYRAMIDS[pyramid]
    g = torch.Generator(device=DEV).manual_seed(N)
    for cin, cout, s in PLANAR:
        x = R.tf32_rna(_randn(g, N, H // s, W // s, cin))
        wt = R.tf32_rna(_randn(g, cout, cin, 3, 3, scale=(9 * cin) ** -0.5))
        shift = _randn(g, cout, scale=0.1)
        wp = ops.pack_conv3d_weight(wt, ops.CONV_PLANAR)
        w64 = R.pack_weight(wt, R.CONV_PLANAR)
        x5 = x.unsqueeze(0)
        y64 = R.epilogue(R.conv3d_ref(x5, w64, R.CONV_PLANAR), None, shift, SLOPE)
        A = R.magnitude(x5, w64, R.CONV_PLANAR)
        xs = x.permute(0, 3, 1, 2)                                  # (N,C,H,W) channels-last
        f0 = _lib.fallback_count()
        for keep in (False, True):
            y = ops.conv2d_planar(xs, wp, cin, cout, shift, SLOPE, ops.TF32, keep_fp32=keep)
            y = y.permute(0, 2, 3, 1).unsqueeze(0)
            assert _is_tf32(y) != keep
            _check(f"planar {pyramid} {cin}->{cout} keep_fp32={keep}", "tma", y, y64, A,
                   0.0 if keep else R.R_TF32, R.epilogue_magnitude(y64, shift))
        assert _lib.fallback_count() == f0
        del y64, A
    for cin, cout, s in P5:
        x = R.tf32_rna(_randn(g, N, H // s, W // s, cin))
        wt = R.tf32_rna(_randn(g, cout, cin, 5, 5, scale=(25 * cin) ** -0.5))
        shift = _randn(g, cout, scale=0.1)
        wp = ops.pack_conv2d_5x5s2_weight(wt)
        w64 = R.pack_weight(wt, R.CONV5X5_S2)
        x5 = x.unsqueeze(0)
        y64 = R.epilogue(R.conv3d_ref(x5, w64, R.CONV5X5_S2), None, shift, SLOPE)
        A = R.magnitude(x5, w64, R.CONV5X5_S2)
        for rnd in (True, False):
            y = ops.conv2d_5x5s2(x.permute(0, 3, 1, 2), wp, shift, SLOPE, round_tf32=rnd)
            y = y.permute(0, 2, 3, 1).unsqueeze(0)
            assert _is_tf32(y) == rnd
            _check(f"5x5s2 {pyramid} {cin}->{cout} round={rnd}", "tma2", y, y64, A,
                   R.R_TF32 if rnd else 0.0, R.epilogue_magnitude(y64, shift))


# ------------------------------------------------------------------------------- backward
# 640x512 training crop, B=1: the stage volumes of test_costreg_backward_vs_oracle scaled up
# (level 0: Cin 8, D 8 at 512x640; level 1: Cin 16, D 32 at 256x320; level 2: Cin 32, D 48)
WGRAD = {   # name: x (layer input) channels, grad_y channels, x dims, stride
    "L0_conv0_8to8": (8, 8, (8, 512, 640), 1),
    "L0_conv1_8to16_s2": (8, 16, (8, 512, 640), 2),
    # transposed conv11 (16 -> 8): the output gradient plays the strided input
    "L0_conv11_T16to8": (8, 16, (8, 512, 640), 2),
    "L1_conv0_16to8": (16, 8, (32, 256, 320), 1),
    "L2_conv0_32to8": (32, 8, (48, 128, 160), 1),
    "L2_conv6_64to64": (64, 64, (6, 16, 20), 1),
}


def _wgrad_fp64(x, gy, stride):
    """dW[tap][a][b] = sum over (b, o) of x[s*o + k - 1, a] gy[o, b], float64, and the same sum
    of |x| |gy|."""
    B, Do, Ho, Wo, _ = gy.shape
    xp = torch.nn.functional.pad(x.double(), (0, 0, 1, 1, 1, 1, 1, 1))
    g64 = gy.double()
    dw = torch.empty(27, x.shape[-1], gy.shape[-1], dtype=torch.float64, device=x.device)
    mag = torch.empty_like(dw)
    s = stride
    for kd in range(3):
        for kh in range(3):
            for kw in range(3):
                xs = xp[:, kd:kd + s * (Do - 1) + 1:s, kh:kh + s * (Ho - 1) + 1:s,
                        kw:kw + s * (Wo - 1) + 1:s]
                t = (kd * 3 + kh) * 3 + kw
                dw[t] = torch.einsum("bdhwa,bdhwc->ac", xs, g64)
                mag[t] = torch.einsum("bdhwa,bdhwc->ac", xs.abs(), g64.abs())
    return dw, mag


@pytest.mark.parametrize("signs", ["mixed", "same"])
@pytest.mark.parametrize("name", list(WGRAD))
def test_conv3d_wgrad_vs_fp64(name, signs):
    """signs='same': non-negative x and gy, every partial sum grows -- the worst case of a long
    sequential fp32 accumulation."""
    ca, cb, dims, stride = WGRAD[name]
    g = torch.Generator(device=DEV).manual_seed(_seed(name))
    x = _randn(g, 1, *dims, ca)
    gy = _randn(g, 1, *R.out_dims(R.CONV, stride, *dims), cb)
    if signs == "same":
        x, gy = x.abs(), gy.abs()
    dw = torch.zeros(27, ca, cb, device=DEV)
    _lib.check(_lib.load().casmvs_conv3d_wgrad(ops._ptr(x), ops._ptr(gy), ops._ptr(dw), 1, ca, cb,
                                               *dims, *gy.shape[1:4], stride, ops._stream()),
               "conv3d_wgrad")
    want, mag = _wgrad_fp64(x, gy, stride)
    ratio = (dw.double() - want).abs() / mag
    need = ratio.max().item()
    t, ab = divmod(int(ratio.argmax()), ca * cb)
    print(f"[fp64] wgrad {name} signs={signs} {tuple(x.shape)}: worst err/sum|x||gy| {need:.3e} "
          f"(eps {EPS['wgrad']:.3e}) at tap {t}, a {ab // cb}, b {ab % cb}")
    assert need <= EPS["wgrad"], (f"wgrad {name} signs={signs}: worst err/sum|x||gy| {need:.3e} "
                                  f"> eps {EPS['wgrad']:.3e} at tap {t}, a {ab // cb}, b {ab % cb}")


DGRAD = {   # name: kind, stride, cin, cout of the FORWARD layer, input dims (level 0 crop)
    "conv0_8to8": (ops.CONV, 1, 8, 8, (8, 512, 640)),
    "conv1_8to16_s2": (ops.CONV, 2, 8, 16, (8, 512, 640)),
    "conv11_T16to8": (ops.CONV_TRANSPOSE, 2, 16, 8, (4, 256, 320)),
}


@pytest.mark.parametrize("precision", [ops.FP32, ops.TF32])
@pytest.mark.parametrize("name", list(DGRAD))
def test_conv3d_dgrad_vs_fp64(name, precision):
    """Data gradient of autograd.Conv3dFn (a forward kernel with re-arranged weights) against
    the float64 adjoint of the layer."""
    kind, stride, cin, cout, dims = DGRAD[name]
    g = torch.Generator(device=DEV).manual_seed(_seed(name))
    x, wt, _, _ = _layer_inputs(g, kind, cin, cout, dims, B=1)
    w64 = R.pack_weight(wt, kind)                                   # (27, cin, cout)
    out = R.out_dims(kind, stride, *dims)
    gy = R.tf32_rna(_randn(g, 1, *out, cout))
    with torch.enable_grad():
        xg = ops.as_volume_view(x).detach().requires_grad_(True)
        y = AG.conv3d(xg, wt, kind, stride, precision)
        y.backward(ops.as_volume_view(gy))
    gx = ops.volume_storage(xg.grad)
    wa = w64.transpose(1, 2)                                        # (27, cout, cin)
    if kind == ops.CONV and stride == 1:
        adj = (wa.flip(0), R.CONV, 1)
        kernel = "tma"
    elif kind == ops.CONV:
        adj = (wa, R.CONV_TRANSPOSE, 2)
        kernel = "tma2"
    else:
        adj = (wa, R.CONV, 2)
        kernel = "tma2"
    want = R.conv3d_ref(gy, *adj)
    A = R.magnitude(gy, *adj)
    tf32 = precision == ops.TF32
    _check(f"dgrad {name} prec={precision} {tuple(x.shape)}", kernel if tf32 else "direct", gx,
           want, A, R.R_TF32 if tf32 else 0.0)
