"""FeatureNet's kernels element by element against float64 (oracle/feature_fp64.py for the
top-down merge and level kernels, oracle/conv3d_fp64.py for every convolution):

  * the whole FeatureNet as the cascade runs it (overlap=True, randomised folded-ABN weights)
    on the cfg2 (640x512, V=3), cfg4 view (1152x864, V=5) and cfg5 view (1920x1056, V=7) image
    batches, in fp32 and tf32.  A fixture records every library call the model makes; each call
    is checked against float64 applied to its own inputs, so errors do not compound, and every
    TF32-rounded store equals tf32_rna of the same call's unrounded output bit for bit;
  * direct calls at ragged shapes: W % 4 != 0 (scalar conv2d_rgb8), h and w not multiples of 16
    (fpn_level tile edges), h w not a multiple of 256 (fpn_merge), odd H and W (5x5 kernel), N > 1.

Bound per element: bound0 + eps A (+ R_TF32 |y| for a TF32-rounded store).  A wgmma call whose
input is not TF32-exact (the 5x5 layers read the planar layers' fp32 outputs in tf32 mode) adds
sum |w| ulp_tf32(x): the operand conversion may truncate or round.  EPS holds, per kernel family,
the largest power of two within 4x of the worst eps needed over this file on an H100 (it prints
them), never more than EPS_CEIL."""
import pytest
import torch

from casmvsnet_pl_b200 import ABN, _lib, ops, synth
from oracle import conv3d_fp64 as R
from oracle import feature_fp64 as FF

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
EPS_CEIL = {"tma": 2.0 ** -14, "tma2": 2.0 ** -14}   # wgmma; every other family: 2^-17
# Worst eps needed over every case of this file, measured on an H100 80GB HBM3 at a 700 W power
# limit; each eps is the largest power of two within 4x of it.  fpn_level's smoothing and the
# 5x5 wgmma layers needed none (the carried merge bound, and the operand term of the tf32 calls,
# cover them): their eps is a nominal 2^-24.
EPS = {
    "rgb8": 2.0 ** -20,          # conv2d_rgb8 / conv2d_rgb8_x4: 3.4e-7
    "direct": 2.0 ** -19,        # planar 3x3 on conv3d_direct (fp32): 5.4e-7
    "5x5_fp32": 2.0 ** -20,      # conv2d_5x5s2_fp32: 4.3e-7
    "merge": 2.0 ** -19,         # fpn_merge, and fpn_level's stored merge: 5.6e-7
    "level": 2.0 ** -24,         # fpn_level's smoothed output: 0
    "tma": 2.0 ** -19,           # planar 3x3 on wgmma (tf32 mode): 4.9e-7
    "tma2": 2.0 ** -24,          # 5x5 stride 2 on wgmma (tf32 mode): 0
}
LOOSE_CEIL = 2.0 ** -8

CONFIGS = {"cfg2": (3, 512, 640), "cfg4_view": (5, 864, 1152), "cfg5_view": (7, 1056, 1920)}
CHAIN = {
    "fp32": {"conv2d_rgb8": 1, "conv2d_planar": 5, "conv2d_5x5s2_fp32": 2, "fpn_merge": 1,
             "fpn_level": 2},
    "tf32": {"conv2d_rgb8": 1, "conv2d_planar": 7, "conv2d_5x5s2": 2, "fpn_merge": 3},
}
RECORDED = ("conv2d_rgb8", "conv2d_planar", "conv2d_5x5s2", "conv2d_5x5s2_fp32", "fpn_merge",
            "fpn_level")


@pytest.fixture
def recorder(monkeypatch):
    """Records (name, args, kwargs, output) of every FeatureNet library call; .orig holds the
    unpatched functions."""
    calls = []
    orig = {n: getattr(ops, n) for n in RECORDED}

    def wrap(name):
        def f(*a, **k):
            out = orig[name](*a, **k)
            calls.append((name, a, k, out))
            return out
        return f
    for n in RECORDED:
        monkeypatch.setattr(ops, n, wrap(n))
    return _Rec(calls, orig)


class _Rec:
    def __init__(self, calls, orig):
        self.calls, self.orig = calls, orig


def _cl(t):
    """logical (N, C, H, W) -> (N, H, W, C) values."""
    return t.permute(0, 2, 3, 1)


def _is_tf32(t):
    return bool((t.contiguous().view(torch.int32) & 0x1FFF).eq(0).all())


def _tf32_ulp(x):
    """Spacing of TF32 values at x: the most the operand conversion (truncation or rounding)
    can move x."""
    ax = x.double().abs()
    e = torch.floor(torch.log2(torch.where(ax > 0, ax, torch.ones_like(ax))))
    return torch.where(ax > 0, torch.exp2(e - 10), torch.zeros_like(ax))


WORST = {}


def _report(tag, fam, rep):
    WORST[fam] = max(WORST.get(fam, 0.0), rep.eps_needed)
    print(f"[fp64] {tag} [{fam}]: {rep.describe()}")
    assert rep.ok, f"{tag} [{fam}]: {rep.describe()}"
    assert rep.loose_share <= LOOSE_CEIL, f"{tag} [{fam}]: loose share {rep.loose_share:.3e}"


def _bit_equal(tag, rounded, unrounded):
    assert _is_tf32(rounded), f"{tag}: rounded store is not TF32-exact"
    a = ops.volume_storage(rounded) if rounded.dim() == 5 else rounded
    want = R.tf32_rna(unrounded.float().contiguous(memory_format=torch.channels_last))
    assert torch.equal(a.contiguous(memory_format=torch.channels_last).view(torch.int32),
                       want.view(torch.int32)), f"{tag}: rounded store != tf32_rna(unrounded)"


# ------------------------------------------------------------------------------- per call
def _conv_check(tag, fam, x5, w64, kind, y5, shift, slope, r, bias_in_acc=False, tf32_in=False):
    """x5 (1, N, H, W, Cin) input, w64 packed float64, y5 (1, N, Ho, Wo, Cout) kernel output;
    one image at a time."""
    for n in range(x5.shape[1]):
        xn = x5[:, n:n + 1]
        acc = R.conv3d_ref(xn, w64, kind)
        y64 = R.epilogue(acc, None, shift, slope)
        A = R.magnitude(xn, w64, kind)
        b0 = torch.zeros_like(y64)
        if bias_in_acc:           # the bias seeds the fma chain: part of the reduction
            A = A + shift.double().abs()
        else:
            b0 = b0 + R.EPI_REL * R.epilogue_magnitude(y64, shift)
        if tf32_in and not _is_tf32(xn):
            b0 = b0 + R.conv3d_ref(_tf32_ulp(xn), w64.abs(), kind)
        rep = FF.check(y5[0, n:n + 1], y64[0], b0[0], A[0], EPS[fam], tf32=r > 0)
        _report(f"{tag} n={n}", fam, rep)


def check_call(rec, name, a, k, out, tag):
    orig = rec.orig[name]
    if name == "conv2d_rgb8":
        x, w, bias, slope = a[:4]
        rnd = k.get("round_tf32", a[4] if len(a) > 4 else False)
        x5 = x.permute(0, 2, 3, 1).unsqueeze(0)
        _conv_check(f"{tag} rgb8 round={rnd}", "rgb8", x5, R.pack_weight(w, R.CONV_PLANAR),
                    R.CONV_PLANAR, _cl(out).unsqueeze(0), bias, slope, R.R_TF32 if rnd else 0.0,
                    bias_in_acc=True)
        if rnd:
            _bit_equal(f"{tag} rgb8", out, orig(x, w, bias, slope, round_tf32=False))
    elif name == "conv2d_planar":
        x, wp, cin, cout = a[:4]
        shift = a[4] if len(a) > 4 else k.get("shift")
        slope = a[5] if len(a) > 5 else k.get("slope", 1.0)
        prec = a[6] if len(a) > 6 else k.get("precision", ops.TF32)
        keep = k.get("keep_fp32", False)
        tf32 = prec == ops.TF32
        w64 = wp.view(27, cin, cout)
        w64 = R.tf32_rna(w64) if tf32 else w64
        rounded = tf32 and not keep
        _conv_check(f"{tag} planar {cin}->{cout} keep={keep}", "tma" if tf32 else "direct",
                    _cl(x).unsqueeze(0), w64.double(), R.CONV_PLANAR, _cl(out).unsqueeze(0),
                    shift, slope, R.R_TF32 if rounded else 0.0, tf32_in=tf32)
        if rounded:
            _bit_equal(f"{tag} planar", out, orig(x, wp, cin, cout, shift, slope, prec,
                                                  keep_fp32=True))
    elif name in ("conv2d_5x5s2", "conv2d_5x5s2_fp32"):
        x, w, shift, slope = a[:4]
        tf32 = name == "conv2d_5x5s2"
        rnd = tf32 and k.get("round_tf32", a[4] if len(a) > 4 else False)
        w64 = R.pack_weight(R.tf32_rna(w.contiguous()) if tf32 else w, R.CONV5X5_S2)
        _conv_check(f"{tag} 5x5s2 {w.shape[1]}->{w.shape[0]} round={rnd}",
                    "tma2" if tf32 else "5x5_fp32", _cl(x).unsqueeze(0), w64, R.CONV5X5_S2,
                    _cl(out).unsqueeze(0), shift, slope, R.R_TF32 if rnd else 0.0, tf32_in=tf32)
        if rnd:
            _bit_equal(f"{tag} 5x5s2", out, orig(x, w, shift, slope, round_tf32=False))
    elif name == "fpn_merge":
        prev, c, lw, lb = a[:4]
        rnd = k.get("round_tf32", a[4] if len(a) > 4 else False)
        for n in range(c.shape[0]):
            pv = None if prev is None else _cl(prev[n:n + 1])
            y64, b0, A = FF.merge_ref(pv, _cl(c[n:n + 1]), lw, lb)
            _report(f"{tag} merge {tuple(c.shape)} prev={prev is not None} round={rnd} n={n}",
                    "merge", FF.check(_cl(out[n:n + 1]), y64, b0, A, EPS["merge"], tf32=rnd))
        if rnd:
            _bit_equal(f"{tag} merge", out, orig(prev, c, lw, lb, round_tf32=False))
    elif name == "fpn_level":
        prev, c, lw, lb, sw, sb = a[:6]
        feat, y = out
        for n in range(c.shape[0]):
            (f64, fb0, fA), (o64, b0, A) = FF.level_ref(_cl(prev[n:n + 1]), _cl(c[n:n + 1]), lw,
                                                        lb, sw, sb)
            t = f"{tag} level {c.shape[1]}->{sw.shape[0]} {tuple(c.shape[2:])} n={n}"
            if feat is not None:
                _report(t + " feat", "merge", FF.check(_cl(feat[n:n + 1]), f64, fb0, fA,
                                                       EPS["merge"]))
            _report(t, "level", FF.check(_cl(y[n:n + 1]), o64, b0, A, EPS["level"]))
            del f64, fb0, fA, o64, b0, A
    else:
        raise AssertionError(name)


# ------------------------------------------------------------------------------- the whole net
def _model(precision):
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    torch.manual_seed(0)
    m = CascadeMVSNet(norm_act=ABN)
    synth.randomize_model_(m, 0)
    return m.eval().to(DEV).set_precision(precision)


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_featurenet_calls_vs_fp64(cfg, precision, recorder):
    N, H, W = CONFIGS[cfg]
    model = _model(precision)
    g = torch.Generator(device=DEV).manual_seed(N)
    imgs = torch.randn(N, 3, H, W, generator=g, device=DEV)
    f0 = _lib.fallback_count()
    feats = model.feature(imgs, overlap=True)
    torch.cuda.synchronize()
    assert _lib.fallback_count() == f0
    assert set(feats) >= {"level_0", "level_1", "level_2"}
    counts = {}
    for name, *_ in recorder.calls:
        counts[name] = counts.get(name, 0) + 1
    assert counts == CHAIN[precision], counts
    calls = list(recorder.calls)
    for name, a, k, out in calls:
        check_call(recorder, name, a, k, out, f"{cfg} {precision}")
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------- ragged shapes
def test_featurenet_kernels_ragged_vs_fp64(recorder):
    g = torch.Generator(device=DEV).manual_seed(7)

    def rn(*s, scale=1.0):
        return torch.randn(*s, generator=g, device=DEV) * scale

    def cl(t):
        return t.contiguous(memory_format=torch.channels_last)
    for H, W in ((37, 141), (9, 1280), (24, 100), (1, 3), (5, 4)):   # W % 4 != 0: scalar kernel
        x = rn(2, 3, H, W)
        wt, b = rn(8, 3, 3, 3, scale=0.3), rn(8, scale=0.2)
        for rnd in (False, True):
            ops.conv2d_rgb8(x, wt, b, 0.01, round_tf32=rnd)
        if W % 4 == 0:                  # an input not 16-byte aligned: the scalar kernel
            buf = torch.empty(x.numel() + 1, device=DEV)
            xs = buf[1:].view(x.shape)
            xs.copy_(x)
            ops.conv2d_rgb8(xs, wt, b, 0.01)
    for N, h, w, clat, cout in ((2, 34, 50, 8, 8), (1, 20, 28, 16, 16), (3, 18, 46, 8, 8),
                                (2, 2, 2, 16, 16), (1, 66, 18, 16, 8)):
        prev, c = cl(rn(N, 32, h // 2, w // 2)), cl(rn(N, clat, h, w))
        lw, lb = rn(32, clat, 1, 1, scale=clat ** -0.5), rn(32, scale=0.5)
        sw, sb = rn(cout, 32, 3, 3, scale=(9 * 32) ** -0.5), rn(cout, scale=0.1)
        ops.fpn_level(prev, c, lw, lb, sw, sb, want_feat=True)
        ops.fpn_level(prev, c, lw, lb, sw, sb, want_feat=False)
    for N, h, w, clat in ((3, 26, 38, 32), (2, 14, 10, 8), (1, 1, 7, 16), (2, 50, 34, 16)):
        c = cl(rn(N, clat, h, w))
        lw, lb = rn(32, clat, 1, 1, scale=clat ** -0.5), rn(32, scale=0.5)
        for rnd in (False, True):
            ops.fpn_merge(None, c, lw, lb, round_tf32=rnd)
            if h % 2 == 0 and w % 2 == 0:
                ops.fpn_merge(cl(rn(N, 32, h // 2, w // 2)), c, lw, lb, round_tf32=rnd)
    for N, H, W, cin, cout in ((2, 37, 53, 8, 16), (3, 19, 33, 16, 32), (1, 1, 1, 8, 16),
                               (2, 64, 80, 16, 32)):
        x = cl(rn(N, cin, H, W))
        wt, sh = rn(cout, cin, 5, 5, scale=(25 * cin) ** -0.5).contiguous(), rn(cout, scale=0.1)
        ops.conv2d_5x5s2_fp32(x, wt, sh, 0.01)
    torch.cuda.synchronize()
    names = {n for n, *_ in recorder.calls}
    assert names == {"conv2d_rgb8", "fpn_level", "fpn_merge", "conv2d_5x5s2_fp32"}
    for name, a, k, out in list(recorder.calls):
        check_call(recorder, name, a, k, out, "ragged")


def test_zz_print_worst():
    """Worst eps needed per family over the file (runs last in file order)."""
    for fam, v in sorted(WORST.items()):
        print(f"[fp64] worst eps needed [{fam}]: {v:.3e} (eps {EPS[fam]:.3e})")
    assert all(e <= EPS_CEIL.get(f, 2.0 ** -17) for f, e in EPS.items())
