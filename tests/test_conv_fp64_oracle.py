"""The float64 convolution reference (oracle/conv3d_fp64.py) and the per-element bound the GPU
tests hold the convolution kernels to: the reference against torch's own float64 convolutions,
the TF32 rounding emulation against hand-written bit patterns, and -- without a GPU -- proof
that the committed tolerances flag the subtle ways a convolution kernel goes wrong."""
import pytest
import torch
import torch.nn.functional as F

from oracle import conv3d_fp64 as R
import test_gpu_conv_fp64 as G
import test_gpu_train_step_fp64 as T

torch.set_default_dtype(torch.float32)


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


def _ncdhw(y):
    return y.permute(0, 4, 1, 2, 3)


def _cl(x):
    return x.permute(0, 2, 3, 4, 1).contiguous()


SHAPES = [(4, 6, 8), (5, 7, 9), (3, 17, 11), (1, 2, 3)]


@pytest.mark.parametrize("dims", SHAPES)
@pytest.mark.parametrize("stride", [1, 2])
def test_conv_matches_torch_conv3d(dims, stride):
    g = torch.Generator().manual_seed(sum(dims) + stride)
    x = torch.randn(2, 8, *dims, generator=g, dtype=torch.float64)
    w = torch.randn(12, 8, 3, 3, 3, generator=g, dtype=torch.float64)
    want = F.conv3d(x, w, None, stride, 1)
    got = _ncdhw(R.conv3d_ref(_cl(x), R.pack_weight(w, R.CONV), R.CONV, stride))
    assert got.shape == want.shape
    assert _rel(got, want) < 1e-12


@pytest.mark.parametrize("dims", SHAPES)
def test_transposed_matches_torch_conv_transpose3d(dims):
    g = torch.Generator().manual_seed(sum(dims))
    x = torch.randn(2, 8, *dims, generator=g, dtype=torch.float64)
    w = torch.randn(8, 4, 3, 3, 3, generator=g, dtype=torch.float64)
    want = F.conv_transpose3d(x, w, None, 2, 1, 1)
    got = _ncdhw(R.conv3d_ref(_cl(x), R.pack_weight(w, R.CONV_TRANSPOSE), R.CONV_TRANSPOSE))
    assert got.shape == want.shape
    assert _rel(got, want) < 1e-12


@pytest.mark.parametrize("hw", [(6, 8), (7, 9), (17, 11), (2, 3)])
def test_planar_and_5x5s2_match_torch_conv2d(hw):
    g = torch.Generator().manual_seed(sum(hw))
    x = torch.randn(2 * 3, 8, *hw, generator=g, dtype=torch.float64)          # B=2 x 3 views
    x_cl = x.permute(0, 2, 3, 1).reshape(2, 3, *hw, 8)
    w3 = torch.randn(12, 8, 3, 3, generator=g, dtype=torch.float64)
    w5 = torch.randn(16, 8, 5, 5, generator=g, dtype=torch.float64)
    for w, kind, stride, pad in ((w3, R.CONV_PLANAR, 1, 1), (w5, R.CONV5X5_S2, 2, 2)):
        want = F.conv2d(x, w, None, stride, pad).permute(0, 2, 3, 1)
        got = R.conv3d_ref(x_cl, R.pack_weight(w, kind), kind)
        assert got.shape == (2, 3) + want.shape[1:]
        assert _rel(got.reshape(want.shape), want) < 1e-12


def test_epilogue_magnitude_and_blocked_layout():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, 5, 6, 8, generator=g, dtype=torch.float64)
    w = torch.randn(27, 8, 4, generator=g, dtype=torch.float64)
    scale = torch.rand(4, generator=g, dtype=torch.float64) - 0.5
    acc = R.conv3d_ref(x, w, R.CONV)
    A = R.magnitude(x, w, R.CONV, scale=scale)
    assert ((acc * scale).abs() <= A * (1 + 1e-12)).all()
    y = R.epilogue(acc, scale, None, 0.01, None)
    v = acc * scale
    assert torch.equal(y, torch.where(v >= 0, v, 0.01 * v))
    assert torch.equal(R.from_blocked(R.to_blocked(x)), x)
    assert torch.equal(R.to_blocked(x)[1, 1, 2, 3, 4], x[1, 2, 3, 4, 4:8])


# ------------------------------------------------------------------------------- tf32_rna
def _bits(v):
    return torch.tensor(v, dtype=torch.int64).to(torch.int32).view(torch.float32)


@pytest.mark.parametrize("src,want", [
    (0x3F800000, 0x3F800000),          # 1.0: already TF32
    (0x3F800FFF, 0x3F800000),          # below half an ulp: down
    (0x3F801000, 0x3F802000),          # tie: away from zero
    (0x3F803000, 0x3F804000),          # tie with an odd kept mantissa: away (not to even)
    (0x3F801001, 0x3F802000),          # above half: up
    (0xBF801000, 0xBF802000),          # negative tie: away from zero (more negative)
    (0xBF800FFF, 0xBF800000),          # negative, below half
    (0x3FFFF000, 0x40000000),          # carry into the exponent
    (0x00000000, 0x00000000),          # +0
    (0x80000000, 0x80000000),          # -0
    (0x00000FFF, 0x00000000),          # subnormal below half an ulp
    (0x00001000, 0x00002000),          # subnormal tie
    (0x807FF000, 0x80800000),          # largest negative subnormal rounds to the smallest normal
    (0x7F7FE000, 0x7F7FE000),          # largest finite TF32
    (0x7F7FFFFF, 0x7F800000),          # largest finite float32 rounds past it: +inf
    (0xFF7FFFFF, 0xFF800000),          # and its negative: -inf
    (0x7F800000, 0x7F800000),          # +inf unchanged
])
def test_tf32_rna_bit_patterns(src, want):
    got = R.tf32_rna(_bits([src]))
    assert got.view(torch.int32).item() == _bits([want]).view(torch.int32).item()


def test_tf32_rna_nan_and_bulk_error():
    nan = _bits([0x7FC00001])
    assert torch.isnan(R.tf32_rna(nan)).all()
    x = torch.randn(100000, generator=torch.Generator().manual_seed(0)) * 1e3
    y = R.tf32_rna(x)
    assert torch.equal(y.view(torch.int32) & 0x1FFF, torch.zeros_like(y, dtype=torch.int32))
    assert ((y.double() - x.double()).abs() <= R.R_TF32 * x.double().abs()).all()


# ------------------------------------------------------------------------------- discrimination
def test_committed_tolerances_within_ceilings():
    assert 0 < G.EPS["tma"] <= G.EPS_CEIL_WGMMA
    assert 0 < G.EPS["tma2"] <= G.EPS_CEIL_WGMMA
    assert 0 < G.EPS["direct"] <= G.EPS_CEIL_FP32
    assert 0 < G.EPS["wgrad"] <= G.EPS_CEIL_FP32


def _layer(cin, cout, dims, seed, B=2):
    """A layer's inputs (TF32-exact, as the GPU tests feed the kernels), its float64 output and
    the float32 output a correct kernel stores (float64 rounded to fp32, then to TF32)."""
    g = torch.Generator().manual_seed(seed)
    x = R.tf32_rna(torch.randn(B, *dims, cin, generator=g)).double()
    w = R.tf32_rna(torch.randn(27, cin, cout, generator=g) * 0.1).double()
    scale = torch.rand(cout, generator=g, dtype=torch.float64) + 0.5
    shift = torch.randn(cout, generator=g, dtype=torch.float64) * 0.1
    return x, w, scale, shift


def _flagged(y, y64, A, extra):
    """At the ceilings, the strictest setting a GPU test may commit, the loosest bound."""
    ok, worst = R.bound_excess(y, y64, A, G.EPS_CEIL_WGMMA, R.R_TF32, extra)
    return not ok


def _stored(y64):
    return R.tf32_rna(y64.float())


def test_correct_output_passes_at_every_tolerance():
    x, w, scale, shift = _layer(16, 16, (6, 20, 12), 3)
    acc = R.conv3d_ref(x, w, R.CONV)
    y64 = R.epilogue(acc, scale, shift, 0.01)
    A = R.magnitude(x, w, R.CONV, scale=scale)
    extra = R.epilogue_magnitude(y64, shift)
    for eps in G.EPS.values():
        assert R.bound_excess(_stored(y64), y64, A, eps, R.R_TF32, extra)[0]
        assert R.bound_excess(y64.float(), y64, A, eps, 0.0, extra)[0]


def test_flags_one_tap_dropped_on_one_slice():
    x, w, scale, shift = _layer(16, 16, (6, 20, 12), 4)
    y64 = R.epilogue(R.conv3d_ref(x, w, R.CONV), scale, shift, 0.01)
    A = R.magnitude(x, w, R.CONV, scale=scale)
    w_drop = w.clone()
    w_drop[13] = 0                                          # centre tap
    bad = y64.clone()
    d = 3                                                   # first slice of a second depth chunk
    bad[:, d] = R.epilogue(R.conv3d_ref(x, w_drop, R.CONV), scale, shift, 0.01)[:, d]
    assert _flagged(_stored(bad), y64, A, R.epilogue_magnitude(y64, shift))
    for tap in (0, 26):                                     # corner taps only: smaller terms
        w_drop = w.clone()
        w_drop[tap] = 0
        bad = y64.clone()
        bad[:, d] = R.epilogue(R.conv3d_ref(x, w_drop, R.CONV), scale, shift, 0.01)[:, d]
        ok, worst = R.bound_excess(_stored(bad), y64, A, G.EPS_CEIL_WGMMA, R.R_TF32,
                                   R.epilogue_magnitude(y64, shift))
        assert not ok and worst["slice"] == d


def test_flags_column_w8_7_shifted_by_one_voxel():
    x, w, scale, shift = _layer(8, 16, (4, 16, 24), 5)
    y64 = R.epilogue(R.conv3d_ref(x, w, R.CONV), scale, shift, 0.01)
    A = R.magnitude(x, w, R.CONV, scale=scale)
    bad = y64.clone()
    for c in range(7, bad.shape[3], 8):
        bad[:, :, :, c] = y64[:, :, :, c - 1]
    ok, worst = R.bound_excess(_stored(bad), y64, A, G.EPS_CEIL_WGMMA, R.R_TF32,
                               R.epilogue_magnitude(y64, shift))
    assert not ok and worst["w8"] == 7


def test_flags_one_k_step_of_one_tap_dropped_cin64():
    x, w, scale, shift = _layer(64, 16, (3, 16, 8), 6, B=1)
    y64 = R.epilogue(R.conv3d_ref(x, w, R.CONV), scale, shift, 0.01)
    A = R.magnitude(x, w, R.CONV, scale=scale)
    extra = R.epilogue_magnitude(y64, shift)
    for tap, k8 in ((13, 7), (0, 0), (22, 3)):
        w_bad = w.clone()
        w_bad[tap, 8 * k8:8 * k8 + 8] = 0                   # one wgmma K step (8 channels)
        bad = R.epilogue(R.conv3d_ref(x, w_bad, R.CONV), scale, shift, 0.01)
        assert _flagged(_stored(bad), y64, A, extra), (tap, k8)


@pytest.mark.parametrize("kind,stride,cin", [(R.CONV, 1, 64), (R.CONV, 2, 32),
                                             (R.CONV_TRANSPOSE, 2, 64)])
def test_flags_cout_chunk_scale_shift_swapped(kind, stride, cin):
    """conv5 / conv6 / conv7 split Cout over blockIdx.y: a CTA reading its neighbour chunk's
    scale and shift (16-channel chunks of 64, 8-channel chunks of 32)."""
    cout = 64 if kind == R.CONV else 32
    chunk = 16 if kind == R.CONV else 8
    x, w, scale, shift = _layer(cin, cout, (3, 6, 10), 7)
    acc = R.conv3d_ref(x, w, kind, stride)
    y64 = R.epilogue(acc, scale, shift, 0.01)
    A = R.magnitude(x, w, kind, stride, scale)
    perm = torch.arange(cout)
    perm[chunk:2 * chunk], perm[2 * chunk:3 * chunk] = (torch.arange(2 * chunk, 3 * chunk),
                                                         torch.arange(chunk, 2 * chunk))
    bad = R.epilogue(acc, scale[perm], shift[perm], 0.01)
    assert _flagged(_stored(bad), y64, A, R.epilogue_magnitude(y64, shift))
    # the same swap with unrounded outputs, at the CUDA-core kernel's ceiling
    ok, _ = R.bound_excess(bad.float(), y64, A, G.EPS_CEIL_FP32, 0.0,
                           R.epilogue_magnitude(y64, shift))
    assert not ok


# ------------------------------------------------------------------------------- data gradient
DGRAD_SHAPES = [   # kind, stride, cin, cout of the forward layer, input dims
    (R.CONV, 1, 8, 12, (4, 6, 8)), (R.CONV, 1, 8, 1, (3, 5, 7)), (R.CONV, 1, 4, 4, (1, 2, 3)),
    (R.CONV, 2, 8, 12, (4, 6, 8)), (R.CONV, 2, 4, 8, (5, 7, 9)), (R.CONV, 2, 4, 1, (2, 3, 4)),
    (R.CONV_TRANSPOSE, 2, 8, 4, (2, 3, 4)), (R.CONV_TRANSPOSE, 2, 4, 1, (3, 2, 5)),
]


def _torch_weight(g, kind, cin, cout, scale=1.0):
    shape = (cout, cin, 3, 3, 3) if kind == R.CONV else (cin, cout, 3, 3, 3)
    return torch.randn(*shape, generator=g, dtype=torch.float64) * scale


@pytest.mark.parametrize("kind,stride,cin,cout,dims", DGRAD_SHAPES)
def test_dgrad_ref_matches_torch_autograd(kind, stride, cin, cout, dims):
    g = torch.Generator().manual_seed(kind * 100 + stride * 10 + cout + sum(dims))
    x = torch.randn(2, cin, *dims, generator=g, dtype=torch.float64, requires_grad=True)
    w = _torch_weight(g, kind, cin, cout)
    y = F.conv3d(x, w, None, stride, 1) if kind == R.CONV else F.conv_transpose3d(x, w, None, 2, 1, 1)
    gy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (want,) = torch.autograd.grad(y, x, gy)
    w64 = R.pack_weight(w, kind)
    got = R.dgrad_ref(_cl(gy), w64, kind, stride, dims)
    assert got.shape == _cl(want).shape
    assert _rel(got, _cl(want)) < 1e-12
    A = R.dgrad_ref(_cl(gy).abs(), w64.abs(), kind, stride, dims)
    assert (got.abs() <= A * (1 + 1e-12)).all()


def test_operand_bias_and_truncation():
    g = torch.Generator().manual_seed(2)
    y64 = torch.randn(4, 5, 6, 7, 8, generator=g, dtype=torch.float64)
    assert R.operand_bias(y64, y64) == 0.0
    assert abs(R.operand_bias(y64 * (1 - 2.0 ** -11), y64) + 2.0 ** -11) < 1e-15
    x = torch.randn(100000, generator=g) * 1e3
    t = R.tf32_trunc(x)
    assert torch.equal(t.view(torch.int32) & 0x1FFF, torch.zeros_like(t, dtype=torch.int32))
    assert (t.abs() <= x.abs()).all() and ((x.double() - t.double()).abs() < 2.0 ** -10 * x.double().abs()).all()
    assert R.operand_bias(t, x.double()) < -2.0 ** -12                 # toward zero, ~0.73 * 2^-11
    assert abs(R.operand_bias(R.tf32_rna(x), x.double())) < 2.0 ** -16  # to nearest: unbiased


def _adjoint_fp32(gy, w, kind, stride, tf32, defect=None, slice_d=None):
    """fp32 restatement of autograd.Conv3dFn's data gradient.  The adjoint layer is built from the
    torch weight w the way Conv3dFn builds it (stride 1: flip the taps, swap the channels, pad a
    Cout = 1 head to 4 zero channels; stride 2: the same weight read as the transposed layer, and
    back), then applied to gy (B, Do, ho, wo, Cout) by conv3d_ref.  In tf32 both operands are
    RNA-rounded and the output is stored TF32-rounded, as the tensor-core kernels do.  defect:
    'unflipped', 'no_transpose', 'tap' (tap 4 of the adjoint dropped on output slice slice_d),
    'pad_values' (the prob head's padding channels filled with copies instead of zeros), 'trunc'
    (gy truncated to TF32 instead of rounded)."""
    gy, w = gy.float(), w.float()
    if tf32:
        gy = R.tf32_trunc(gy) if defect == "trunc" else R.tf32_rna(gy)
        w = R.tf32_rna(w)
    if kind == R.CONV and stride == 1:
        wt = w if defect == "unflipped" else w.flip(2, 3, 4)
        if defect != "no_transpose":
            wt = wt.transpose(0, 1)                                # (Cin, Cout, 3, 3, 3)
        pad = -gy.shape[-1] % 4
        if pad and defect == "pad_values":
            gy = torch.cat([gy] + [gy[..., :1]] * pad, -1)
            wt = torch.cat([wt] + [wt[:, :1]] * pad, 1)
        elif pad:
            gy = F.pad(gy, (0, pad))
            wt = F.pad(wt, (0, 0, 0, 0, 0, 0, 0, pad))
        wa, k, s = R.pack_weight(wt, R.CONV), R.CONV, 1
    elif kind == R.CONV:
        wa, k, s = R.pack_weight(w, R.CONV_TRANSPOSE), R.CONV_TRANSPOSE, 2
    else:
        wa, k, s = R.pack_weight(w, R.CONV), R.CONV, 2
    out = R.conv3d_ref(gy, wa, k, s)
    if defect == "tap":
        wd = wa.clone()
        wd[4] = 0                                  # (kd, kh, kw) = (0, 1, 1): reaches odd slices too
        out[:, slice_d] = R.conv3d_ref(gy, wd, k, s)[:, slice_d]
    out = out.float()
    return R.tf32_rna(out) if tf32 else out


def _dgrad_case(kind, stride, cin, cout, dims, seed):
    """A layer's torch weight and an fp32 output gradient that is not TF32-exact (as the norm-act
    backward produces it), with the float64 data gradient and its magnitude for both precisions."""
    g = torch.Generator().manual_seed(seed)
    w = _torch_weight(g, kind, cin, cout, (27 * cin) ** -0.5).float()
    gy = torch.randn(2, *R.out_dims(kind, stride, *dims), cout, generator=g)
    assert not T._is_tf32(gy)
    ref = {}
    for tf32 in (False, True):
        w64 = R.pack_weight(R.tf32_rna(w) if tf32 else w, kind)
        ref[tf32] = (R.dgrad_ref(gy, w64, kind, stride, dims),
                     R.dgrad_ref(gy.abs(), w64.abs(), kind, stride, dims))
    return w, gy, ref


def _report(got, ref, kind, stride, tf32):
    """T.conv_report of an adjoint restatement, as the GPU test runs it on a recorded call."""
    want, A = ref[tf32]
    kernel = ("tma" if kind == R.CONV and stride == 1 else "tma2") if tf32 else "direct"
    return T.conv_report(got, want, A, kernel, R.R_TF32 if tf32 else 0.0,
                         T.R_OP if tf32 else 0.0)


@pytest.mark.parametrize("kind,stride,cin,cout,dims", [
    (R.CONV, 1, 16, 8, (4, 12, 10)), (R.CONV, 1, 8, 1, (4, 12, 10)), (R.CONV, 2, 8, 16, (4, 12, 10)),
    (R.CONV_TRANSPOSE, 2, 16, 8, (2, 6, 5))])
def test_clean_adjoint_restatement_passes(kind, stride, cin, cout, dims):
    w, gy, ref = _dgrad_case(kind, stride, cin, cout, dims, 21)
    for tf32 in (False, True):
        ok, bias_ok, worst, need, bias = _report(_adjoint_fp32(gy, w, kind, stride, tf32), ref,
                                                 kind, stride, tf32)
        assert ok and bias_ok, (tf32, worst, bias)


def _assert_located(worst, got, ref, tf32):
    """The report points at a voxel whose error really is outside the bound."""
    want, A = ref[tf32]
    at = worst["at"]
    assert worst["got"] == float(got[at]) and worst["want"] == float(want[at])
    assert abs(worst["got"] - worst["want"]) > (T.EPS["tma"] + T.R_OP) * float(A[at])


@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("defect,layer", [
    ("unflipped", (R.CONV, 1, 16, 8, (4, 12, 10))),
    ("no_transpose", (R.CONV, 1, 16, 16, (4, 12, 10))),
    ("pad_values", (R.CONV, 1, 8, 1, (4, 12, 10))),
])
def test_flags_wrong_adjoint_weight(defect, layer, tf32):
    kind, stride, cin, cout, dims = layer
    w, gy, ref = _dgrad_case(kind, stride, cin, cout, dims, 22)
    got = _adjoint_fp32(gy, w, kind, stride, tf32, defect)
    ok, _, worst, need, _ = _report(got, ref, kind, stride, tf32)
    assert not ok, (defect, need)
    _assert_located(worst, got, ref, tf32)


@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("kind,stride,cin,cout,dims", [
    (R.CONV, 1, 16, 8, (6, 12, 10)), (R.CONV, 2, 8, 16, (6, 12, 10)),
    (R.CONV_TRANSPOSE, 2, 16, 8, (5, 6, 5))])
def test_flags_one_adjoint_tap_dropped_on_one_slice(kind, stride, cin, cout, dims, tf32):
    w, gy, ref = _dgrad_case(kind, stride, cin, cout, dims, 23)
    d = 3
    got = _adjoint_fp32(gy, w, kind, stride, tf32, "tap", slice_d=d)
    ok, _, worst, _, _ = _report(got, ref, kind, stride, tf32)
    assert not ok and worst["slice"] == d
    _assert_located(worst, got, ref, tf32)


@pytest.mark.parametrize("kind,stride,cin,cout,dims", [
    (R.CONV, 1, 16, 8, (4, 12, 10)), (R.CONV, 2, 8, 16, (4, 12, 10)),
    (R.CONV_TRANSPOSE, 2, 16, 8, (2, 6, 5))])
def test_flags_truncated_operand_by_its_bias(kind, stride, cin, cout, dims):
    """An operand truncated to TF32 stays within the per-element bound (its error is below an ulp
    of TF32) but not within the bias check, which names its size and direction."""
    w, gy, ref = _dgrad_case(kind, stride, cin, cout, dims, 24)
    ok, bias_ok, _, _, bias = _report(_adjoint_fp32(gy, w, kind, stride, True, "trunc"), ref,
                                      kind, stride, True)
    assert not bias_ok and bias < -4 * T.BIAS_MAX, bias
    _, bias_ok, _, _, bias = _report(_adjoint_fp32(gy, w, kind, stride, True), ref, kind, stride, True)
    assert bias_ok and abs(bias) < T.BIAS_MAX / 4, bias
