"""CPU checks of the float64 FeatureNet / regression / hypothesis oracles (oracle/feature_fp64.py,
oracle/regress_fp64.py), no GPU needed:

  * the float64 references equal torch's float64 F.interpolate(align_corners=True), F.conv2d,
    softmax and autograd to 1e-12;
  * an unfused fp32 restatement of each kernel's arithmetic (csrc/fpn.cu, csrc/regress.cu,
    regress_bwd_kernel) passes the bound at every element;
  * the same restatement with one injected defect fails it, and the report points at the
    defect's location (channel group, tile column, plane, batch item)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import feature_fp64 as FF
from oracle import regress_fp64 as RG
from oracle.conv3d_fp64 import tf32_rna

EPS = 2.0 ** -17                 # the fp32 CUDA-core ceiling of the GPU checks
F32 = torch.float32


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------- fp32 restatements
def _axis_f32(n_out, n_in, defect=None, clamp_hi=True):
    if defect == "scale_hi_over_h":
        s = torch.tensor(n_in, dtype=F32) / torch.tensor(n_out, dtype=F32)
    else:
        s = (torch.tensor(n_in - 1, dtype=F32) / torch.tensor(n_out - 1, dtype=F32)
             if n_in > 1 else torch.tensor(0.0))
    f = s * torch.arange(n_out, dtype=F32)
    i0 = f.trunc().long().clamp(max=n_in - 1)
    i1 = (i0 + 1).clamp(max=n_in - 1) if clamp_hi else i0 + 1
    return i0, i1, f - i0.to(F32)


def up_f32(prev, defect=None):
    """fpn_merge / fpn_level / hypotheses_kernel bilinear blend, float32, one rounding per
    operation.  defect 'unclamped': the right tap x0 + 1 is not clamped and reads the next
    texel in memory: the first of the next row, or past the end of the image (NaN here)."""
    N, hi, wi, C = prev.shape
    h, w = 2 * hi, 2 * wi
    y0, y1, ly = _axis_f32(h, hi, defect)
    x0, x1, lx = _axis_f32(w, wi, defect, clamp_hi=defect != "unclamped")
    flat = torch.cat([prev.reshape(N, hi * wi, C), torch.full((N, wi, C), float("nan"))], 1)
    ly, lx = ly.view(1, h, 1, 1), lx.view(1, 1, w, 1)

    def tap(yy, xx):
        return flat[:, (yy.view(h, 1) * wi + xx.view(1, w)).reshape(-1)].view(N, h, w, C)
    w00, w01 = (1 - ly) * (1 - lx), (1 - ly) * lx
    w10, w11 = ly * (1 - lx), ly * lx
    return ((tap(y0, x0) * w00 + tap(y0, x1) * w01) + tap(y1, x0) * w10) + tap(y1, x1) * w11


def merge_f32(prev, c, lw, lb, defect=None):
    """fpn_merge: (blend) + bias, then the lateral products one channel at a time."""
    N, h, w, clat = c.shape
    v = lb.view(1, 1, 1, -1).expand(N, h, w, 32).clone()
    if defect == "bias_group3":
        v[..., 24:] = 0
    if prev is not None:
        v = up_f32(prev, defect) + v
    for ci in range(clat - (4 if defect == "lateral_short" else 0)):
        v = v + c[..., ci:ci + 1] * lw[:, ci].view(1, 1, 1, 32)
    return v


def conv3x3_f32(x, wt, bias, pad_cols=None):
    """3x3 pad-1 Conv2d, bias first, taps (ci, ky, kx) or (ky, kx, ci) one at a time:
    x (N, H, W, Cin) -> (N, H, W, Cout).  pad_cols: (mod, rem) -- output pixels with
    x % mod == rem see their right neighbour column as zero."""
    N, H, W, cin = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    if pad_cols is not None:
        mod, rem = pad_cols
        xz = xp.clone()
        cols = torch.arange(W + 2)
        xz[:, :, (cols - 1) % mod == (rem + 1) % mod] = 0
    acc = bias.view(1, 1, 1, -1).expand(N, H, W, wt.shape[0]).clone()
    for ci in range(cin):
        for ky in range(3):
            for kx in range(3):
                t = xp[:, ky:ky + H, kx:kx + W, ci:ci + 1]
                if pad_cols is not None and kx == 2:
                    sel = (torch.arange(W) % mod == rem).view(1, 1, W, 1)
                    t = torch.where(sel, xz[:, ky:ky + H, kx:kx + W, ci:ci + 1], t)
                acc = acc + t * wt[:, ci, ky, kx].view(1, 1, 1, -1)
    return acc


def rgb8_f32(x, wt, bias, slope, round_tf32=False, defect=None):
    """conv2d_rgb8: planar (N, 3, H, W) -> (N, H, W, 8); defect 'x4_in5': the x4 kernel's right
    neighbour in[5] read as zero (pixels x % 4 == 3)."""
    acc = conv3x3_f32(x.permute(0, 2, 3, 1), wt, bias, (4, 3) if defect == "x4_in5" else None)
    y = torch.where(acc >= 0, acc, acc * slope)
    return tf32_rna(y.contiguous()) if round_tf32 else y


def level_f32(prev, c, lw, lb, sw, sb, defect=None):
    feat = merge_f32(prev, c, lw, lb, defect)
    return feat, conv3x3_f32(feat, sw, sb, (16, 15) if defect == "halo_col" else None)


def _cascade16(terms):
    a0 = torch.zeros_like(terms[0])
    a1 = torch.zeros_like(a0)
    for i, t in enumerate(terms):
        a0 = a0 + t
        if i % 16 == 15:
            a1, a0 = a1 + a0, torch.zeros_like(a0)
    return a0 + a1


def _exp_f32(t):
    return t.double().exp().to(F32)                  # correctly rounded exp of the fp32 argument


def regress_f32(l, dv, input_is_prob=False, defect=None):
    """regress_kernel in float32: -> depth, conf, index, prob.  dv (B, D, h, w)."""
    B, D, h, w = l.shape
    if input_is_prob:
        p = l.clone()
    else:
        e = _exp_f32(l - l.amax(1, keepdim=True))
        den = torch.zeros(B, h, w)
        for d in range(D - (1 if defect == "denom_short" else 0)):
            den = den + e[:, d]
        p = e / den.unsqueeze(1)
    hp = dv.clone()
    if defect == "plane_hyp":
        hp[:, D // 2] = dv[:, D // 2 - 1]
    depth = _cascade16([p[:, d] * hp[:, d] for d in range(D)])
    fidx = _cascade16([p[:, d] * float(d) for d in range(D)])
    idx = (fidx.round() if defect == "index_round" else fidx.trunc()).clamp(0, D - 1).long()
    lo = -2 if defect == "conf_window" else -1
    conf = torch.zeros(B, h, w)
    for k in range(lo, lo + 4):
        d = idx + k
        inside = (d >= 0) & (d < D)
        conf = conf + torch.where(inside, p.gather(1, d.clamp(0, D - 1).unsqueeze(1))[:, 0], 0.0)
    return depth, conf, idx, p


def regress_bwd_f32(l, dv, gd, defect_plane=None):
    B, D, h, w = l.shape
    e = _exp_f32(l - l.amax(1, keepdim=True))
    den = torch.zeros(B, h, w)
    num = torch.zeros(B, h, w)
    for d in range(D):
        den = den + e[:, d]
        num = (e[:, d].double() * dv[:, d].double() + num.double()).to(F32)       # fmaf
    depth = num / den
    g = gd / den
    out = torch.empty_like(l)
    for d in range(D):
        diff = depth - dv[:, d] if d == defect_plane else dv[:, d] - depth
        out[:, d] = e[:, d] * diff * g
    return out


def hypotheses_f32(cur, D, step, upsample, defect=None):
    """hypotheses_kernel: cur (B, h/2, w/2) (upsample) or (B, h, w); step float or (B,)."""
    c = up_f32(cur.unsqueeze(-1))[..., 0] if upsample else cur
    B = c.shape[0]
    s = torch.as_tensor(step, dtype=F32).reshape(-1).expand(B).view(B, 1, 1)
    half = (D * s) if defect == "half_D" else torch.tensor(float(D) * 0.5, dtype=F32) * s
    first = torch.clamp_min(c - half, RG.THRESH)
    out = []
    for d in range(D):
        sd = s * torch.tensor(float(d), dtype=F32)
        out.append(torch.clamp_min((c - half) + sd, RG.THRESH) if defect == "clamp_after"
                   else first + sd)
    return torch.stack(out, 1)


# ------------------------------------------------------------------------------- inputs
def _fpn_inputs(seed, N=2, h=20, w=40, clat=16, cout=8):
    g = _gen(seed)
    prev = torch.randn(N, h // 2, w // 2, 32, generator=g)
    c = torch.randn(N, h, w, clat, generator=g)
    lw = torch.randn(32, clat, generator=g) * clat ** -0.5
    lb = torch.randn(32, generator=g) * 0.5
    sw = torch.randn(cout, 32, 3, 3, generator=g) * (9 * 32) ** -0.5
    sb = torch.randn(cout, generator=g) * 0.1
    return prev, c, lw, lb, sw, sb


def _k3_inputs(seed, B=2, D=32, h=9, w=37, scale=4.0, ladder=False):
    g = _gen(seed)
    l = torch.randn(B, D, h, w, generator=g) * scale
    if ladder:          # per-item ladder, materialised like ops.Ladder: product, then sum
        first = torch.tensor([425.0, 431.5]).view(B, 1, 1, 1)
        step = torch.tensor([2.65, 3.1]).view(B, 1, 1, 1)
        dv = (first + step * torch.arange(D, dtype=F32).view(1, D, 1, 1)).expand(B, D, h, w)
        return l, dv.contiguous(), first, step
    dv = torch.rand(B, D, h, w, generator=g) * 500 + 400
    return l, dv


# ------------------------------------------------------------------------------- float64 references
def test_upsample_matches_interpolate():
    g = _gen(1)
    for hi, wi in ((1, 1), (1, 7), (5, 3), (10, 17), (64, 80)):
        prev = torch.randn(2, hi, wi, 5, generator=g)
        up, b0, M = FF.upsample2x(prev)
        want = F.interpolate(prev.double().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear",
                             align_corners=True).permute(0, 2, 3, 1)
        assert (up - want).abs().max() < 1e-12
        assert bool((b0 >= 0).all()) and bool((M >= up.abs() - 1e-12).all())


def test_merge_and_level_match_conv2d():
    prev, c, lw, lb, sw, sb = _fpn_inputs(2, w=38)
    (feat, _, fA), (out, _, A) = FF.level_ref(prev, c, lw, lb, sw, sb)
    up = F.interpolate(prev.double().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear",
                       align_corners=True)
    lat = F.conv2d(c.double().permute(0, 3, 1, 2), lw.double().view(32, -1, 1, 1), lb.double())
    f = up + lat
    o = F.conv2d(f, sw.double(), sb.double(), padding=1)
    assert (feat - f.permute(0, 2, 3, 1)).abs().max() < 1e-12
    assert (out - o.permute(0, 2, 3, 1)).abs().max() < 1e-12
    lat_only, b0, _ = FF.merge_ref(None, c, lw, lb)
    assert (lat_only - lat.permute(0, 2, 3, 1)).abs().max() < 1e-12 and float(b0.abs().max()) == 0
    assert bool((A >= out.abs() - 1e-12).all()) and bool((fA >= feat.abs() - 1e-12).all())


def test_regress_references_match_torch():
    l, dv = _k3_inputs(3, scale=30.0)
    ref = RG.regress_ref(l, dv)
    p = torch.softmax(l.double(), 1)
    assert (ref["p"] - p).abs().max() < 1e-12
    assert ((ref["depth"] - (p * dv.double()).sum(1)).abs() / ref["depth"].abs()).max() < 1e-12
    dd = torch.arange(l.shape[1], dtype=torch.float64).view(1, -1, 1, 1)
    assert (ref["fidx"] - (p * dd).sum(1)).abs().max() < 1e-12
    vec = dv[0, :, 0, 0].contiguous()
    rv = RG.regress_ref(l, vec)
    assert ((rv["depth"] - (p * vec.double().view(1, -1, 1, 1)).sum(1)).abs()).max() < 1e-9
    gd = torch.randn(l.shape[0], *l.shape[2:], generator=_gen(4))
    lg = l.double().requires_grad_(True)
    with torch.enable_grad():
        (torch.softmax(lg, 1) * dv.double()).sum(1).mul(gd.double()).sum().backward()
    g64, _, A = RG.regress_bwd_ref(l, dv, gd)
    assert ((g64 - lg.grad).abs() - 1e-12 * A).max() <= 0


def test_hypotheses_reference_matches_interpolate():
    g = _gen(5)
    cur = torch.rand(2, 6, 9, generator=g) * 50 + 30
    out, bound, clamped = RG.hypotheses_ref(cur, 32, 2.65, True)
    up = F.interpolate(cur.double().unsqueeze(1), scale_factor=2, mode="bilinear",
                       align_corners=True)
    want = (up - 16 * 2.65).clamp_min(RG.THRESH) + 2.65 * torch.arange(32).double().view(1, -1, 1, 1)
    assert (out - want).abs().max() < 1e-12
    assert bool(clamped.any()) and bool((~clamped).any())
    uni, _ = RG.uniform_ref(425.0, 10.6, 2, 48, 3, 4)
    assert (uni - (425.0 + 10.6 * torch.arange(48).double()).view(1, -1, 1, 1)).abs().max() < 1e-12


# ------------------------------------------------------------------------------- restatements pass
def _assert_ok(rep, what):
    print(f"[oracle] {what}: {rep.describe()}")
    assert rep.ok, f"{what}: {rep.describe()}"


def test_fpn_restatements_within_bound():
    prev, c, lw, lb, sw, sb = _fpn_inputs(6)
    (feat64, fb0, fA), (out64, b0, A) = FF.level_ref(prev, c, lw, lb, sw, sb)
    feat, out = level_f32(prev, c, lw, lb, sw, sb)
    _assert_ok(FF.check(feat, feat64, fb0, fA, EPS), "merge")
    _assert_ok(FF.check(tf32_rna(feat), feat64, fb0, fA, EPS, tf32=True), "merge tf32")
    _assert_ok(FF.check(out, out64, b0, A, EPS), "level")
    y64, yb0, yA = FF.merge_ref(None, c, lw, lb)
    _assert_ok(FF.check(merge_f32(None, c, lw, lb), y64, yb0, yA, EPS), "lateral only")


def _rgb8_ref(x, wt, bias, slope):
    from oracle import conv3d_fp64 as R
    x5 = x.permute(0, 2, 3, 1).unsqueeze(0)
    w64 = R.pack_weight(wt, R.CONV_PLANAR)
    acc = R.conv3d_ref(x5, w64, R.CONV_PLANAR)[0]
    y64 = R.epilogue(acc, None, bias, slope)
    A = R.magnitude(x5, w64, R.CONV_PLANAR)[0] + bias.double().abs()
    return y64, torch.zeros_like(y64), A


def _rgb8_inputs(seed, H=11, W=36):
    g = _gen(seed)
    return (torch.randn(2, 3, H, W, generator=g), torch.randn(8, 3, 3, 3, generator=g) * 0.3,
            torch.randn(8, generator=g) * 0.2, 0.01)


def test_rgb8_restatement_within_bound():
    x, wt, b, slope = _rgb8_inputs(7)
    y64, b0, A = _rgb8_ref(x, wt, b, slope)
    for rnd in (False, True):
        _assert_ok(FF.check(rgb8_f32(x, wt, b, slope, rnd), y64, b0, A, EPS, tf32=rnd),
                   f"rgb8 round={rnd}")


@pytest.mark.parametrize("is_prob", [False, True])
@pytest.mark.parametrize("D", [8, 48])
def test_regress_restatement_within_bound(D, is_prob):
    l, dv = _k3_inputs(8 + D, D=D, scale=30.0 if D == 8 else 4.0)
    if is_prob:
        l = torch.softmax(l, 1)
    depth, conf, idx, p = regress_f32(l, dv, is_prob)
    reps = RG.check_regress(l, dv, depth, conf, idx, None if is_prob else p, is_prob, EPS)
    for k in ("prob", "depth", "conf"):
        if k in reps:
            _assert_ok(reps[k], f"K3 D={D} prob_in={is_prob} {k}")
    assert reps["index"][0] == 0, reps["index"]


def test_regress_bwd_and_hypotheses_restatements_within_bound():
    l, dv = _k3_inputs(9, D=32)
    gd = torch.randn(2, 9, 37, generator=_gen(10))
    g64, b0, A = RG.regress_bwd_ref(l, dv, gd)
    _assert_ok(FF.check(regress_bwd_f32(l, dv, gd), g64, b0, A, EPS, names=("b", "d", "y", "x")),
               "K3 backward")
    cur = torch.rand(2, 10, 19, generator=_gen(11)) * 60 + 20
    for step, up in ((2.65, True), (torch.tensor([2.65, 5.3]), True), (1.5, False)):
        c = cur if up else cur[:, :, :18]
        out64, bound, clamped = RG.hypotheses_ref(c, 32, step, up)
        got = hypotheses_f32(c, 32, step, up)
        _assert_ok(FF.check(got, out64, bound, torch.zeros_like(bound), EPS,
                            names=("b", "d", "y", "x")), f"K4 upsample={up}")
        assert bool(clamped.any())
        assert bool((got[:, 0][clamped] == RG.THRESH).all())


# ------------------------------------------------------------------------------- defects fail
def _fails(rep, what):
    print(f"[oracle] defect {what}: {rep.describe()}")
    assert not rep.ok, f"defect {what} passed the bound: {rep.describe()}"
    return dict(zip(rep.names, rep.worst["at"]))


def test_defect_upsample_scale():
    prev, c, lw, lb, _, _ = _fpn_inputs(12)
    y64, b0, A = FF.merge_ref(prev, c, lw, lb)
    at = _fails(FF.check(merge_f32(prev, c, lw, lb, "scale_hi_over_h"), y64, b0, A, EPS),
                "upsample scale hi/h")
    assert at["y"] > 0 or at["x"] > 0


def test_defect_right_edge_unclamped():
    """At x = w - 1 the kernels' position is exactly wi - 1, so the unclamped tap has weight 0:
    it shows where the memory past the image holds a NaN (0 * NaN)."""
    prev, c, lw, lb, _, _ = _fpn_inputs(13)
    y64, b0, A = FF.merge_ref(prev, c, lw, lb)
    assert FF.check(merge_f32(prev, c, lw, lb), y64, b0, A, EPS).ok
    at = _fails(FF.check(merge_f32(prev, c, lw, lb, "unclamped"), y64, b0, A, EPS),
                "right-edge tap unclamped")
    assert at["x"] == c.shape[2] - 1


@pytest.mark.parametrize("defect,lo,hi", [("bias_group3", 24, 32), ("lateral_short", 0, 32)])
def test_defect_lateral(defect, lo, hi):
    prev, c, lw, lb, _, _ = _fpn_inputs(14)
    y64, b0, A = FF.merge_ref(prev, c, lw, lb)
    at = _fails(FF.check(merge_f32(prev, c, lw, lb, defect), y64, b0, A, EPS), defect)
    assert lo <= at["c"] < hi


def test_defect_level_halo_column():
    prev, c, lw, lb, sw, sb = _fpn_inputs(15, w=64)
    _, (out64, b0, A) = FF.level_ref(prev, c, lw, lb, sw, sb)
    _, out = level_f32(prev, c, lw, lb, sw, sb, "halo_col")
    at = _fails(FF.check(out, out64, b0, A, EPS), "fpn_level halo column zeroed")
    assert at["x"] % 16 == 15


def test_defect_rgb8_x4_right_neighbour():
    x, wt, b, slope = _rgb8_inputs(16)
    y64, b0, A = _rgb8_ref(x, wt, b, slope)
    at = _fails(FF.check(rgb8_f32(x, wt, b, slope, defect="x4_in5"), y64, b0, A, EPS),
                "rgb8_x4 in[5] zeroed")
    assert at["x"] % 4 == 3


@pytest.mark.parametrize("defect", ["conf_window", "index_round", "denom_short", "plane_hyp"])
def test_defect_regress(defect):
    D = 32
    l, dv = _k3_inputs(17, D=D)
    depth, conf, idx, p = regress_f32(l, dv, defect=defect)
    reps = RG.check_regress(l, dv, depth, conf, idx, p, False, EPS)
    if defect == "index_round":
        wrong, amb, first = reps["index"]
        print(f"[oracle] defect {defect}: {wrong} wrong indices ({amb} ambiguous), first at {first}")
        assert wrong > 0
        return
    key = {"conf_window": "conf", "denom_short": "prob", "plane_hyp": "depth"}[defect]
    _fails(reps[key], f"{defect} ({key})")
    if defect == "denom_short":
        assert not reps["depth"].ok


def test_defect_ladder_step_of_item_0():
    l, dv, first, step = _k3_inputs(18, D=48, ladder=True)
    bad = dv.clone()
    bad[1] = first[1] + step[0] * torch.arange(48, dtype=F32).view(48, 1, 1)
    depth, conf, idx, _ = regress_f32(l, bad)
    at = _fails(RG.check_regress(l, dv, depth, conf, idx, None, False, EPS)["depth"],
                "item 1 with item 0's step")
    assert at["b"] == 1


def test_defect_bwd_sign():
    l, dv = _k3_inputs(19, D=32)
    gd = torch.randn(2, 9, 37, generator=_gen(20))
    g64, b0, A = RG.regress_bwd_ref(l, dv, gd)
    at = _fails(FF.check(regress_bwd_f32(l, dv, gd, defect_plane=5), g64, b0, A, EPS,
                         names=("b", "d", "y", "x")), "backward sign at plane 5")
    assert at["d"] == 5


@pytest.mark.parametrize("defect", ["clamp_after", "half_D"])
def test_defect_hypotheses(defect):
    cur = torch.rand(2, 10, 19, generator=_gen(21)) * 60 + 20
    out64, bound, clamped = RG.hypotheses_ref(cur, 32, 2.65, True)
    assert bool(clamped.any())
    got = hypotheses_f32(cur, 32, 2.65, True, defect)
    at = _fails(FF.check(got, out64, bound, torch.zeros_like(bound), EPS,
                         names=("b", "d", "y", "x")), f"K4 {defect}")
    if defect == "clamp_after":
        assert bool(clamped[at["b"], at["y"], at["x"]]) and at["d"] > 0
