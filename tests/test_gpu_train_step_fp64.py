"""Every CostRegNet convolution of real training steps element by element against float64, in
fp32 and tf32, together with the cost-volume (K1) and depth-regression (K3) calls of the same
steps.

The model is built by train.build_model and stepped by train.Trainer.train_step on synthetic
samples with about 20 % of the depth mask missing.  autograd.Conv3dFn, WarpCostFn and RegressFn
are wrapped so that every call's inputs and outputs are cloned when the call is made (the
norm-act overwrites its input in place), with the casmvs_fallback_count difference around each
Conv3dFn launch, which tells which kernel ran.  Each call is then checked against float64
applied to its own recorded inputs, so errors do not compound:

  * forward y against conv3d_ref(x, w64), data gradient gx against dgrad_ref(gy, w64) (the
    float64 vector-Jacobian product of the layer, not a re-arranged weight), weight gradient
    against wgrad_ref of the operand the forward kernel read;
  * K1 and its backward by warp_cost_fp64, K3 and its backward by regress_fp64, at the eps of
    their own files.

w64 is the weight the kernel multiplies: RNA-rounded for a tensor-core call, fp32 for the
CUDA-core kernel.  Per element, |y - y64| <= eps_k A + r_op A + r |y64| + tiny, with eps_k the
committed eps of the kernel that ran (test_gpu_conv_fp64.EPS), r = R_TF32 where the output is
stored TF32-rounded, and r_op = R_OP where a tensor-core call received an operand that is not
TF32-exact: autograd.Conv3dFn rounds it to nearest first, an error of at most half an ulp.  For
those calls the relative bias sum (y - y64) sign(y64) / sum |y64| must stay within BIAS_MAX.
wgmma itself truncates a non-TF32 operand, which gives a bias of about -3.5e-4 (0.73 * 2^-11);
this check fails by a factor of six if the rounding is dropped.

Each step makes 33 forward, 33 data-gradient and 33 weight-gradient calls (11 layers at each
of 3 levels).  In tf32, the data gradients without a tensor-core kernel are asserted by name:
the three prob heads (Cout = 1, padded to 4 input channels) and, with one group, the middle
level's conv0 (8 -> 16)."""
import inspect
import os

import pytest
import torch

import test_gpu_conv_fp64 as CONV_T
import test_gpu_regress_fp64 as REG_T
import test_gpu_warp_cost_fp64 as K1_T
from casmvsnet_pl_b200 import _lib, ops, synth, train
from casmvsnet_pl_b200 import autograd as AG
from oracle import conv3d_fp64 as R
from oracle import conv3d_wgrad_fp64 as WG
from oracle import regress_fp64 as RG
from oracle import warp_cost_fp64 as W

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
EPS = CONV_T.EPS                 # tma, tma2, direct
# the weight gradient's eps of test_gpu_conv_fp64, which holds for same-sign operands: conv0's
# input is the non-negative variance volume, and most of every other input is a LeakyReLU output
EPS_WGRAD = CONV_T.EPS["wgrad"]
EPS_K1 = K1_T.EPS                # staged, gather, bwd
EPS_K3 = REG_T.EPS               # k3, k3_bwd
R_OP = 2.0 ** -11                # RNA rounding of a tensor-core operand: half an ulp of TF32
BIAS_MAX = 2.0 ** -14            # |operand_bias| of a call with a rounded operand

LAYERS = ("conv0", "conv1", "conv2", "conv3", "conv4", "conv5", "conv6", "conv7", "conv9",
          "conv11", "prob")
LEVELS = (2, 1, 0)               # the order the cascade runs its stages
KINDS = {n: (ops.CONV_TRANSPOSE, 2) if n in ("conv7", "conv9", "conv11") else
         (ops.CONV, 2) if n in ("conv1", "conv3", "conv5") else (ops.CONV, 1) for n in LAYERS}

CASES = {   # name: data, W, H, B, precision, num_groups, one step and SGD update first, deterministic
    "dtu_fp32": ("dtu", 640, 512, 1, "fp32", 1, False, False),
    "dtu_tf32_after_update": ("dtu", 640, 512, 1, "tf32", 1, True, False),
    "dtu_tf32_b2": ("dtu", 640, 512, 2, "tf32", 1, False, False),
    "dtu_tf32_g8": ("dtu", 640, 512, 1, "tf32", 8, False, False),
    "blendedmvs_fp32": ("blendedmvs", 768, 576, 1, "fp32", 1, False, False),
    "blendedmvs_tf32": ("blendedmvs", 768, 576, 1, "tf32", 1, False, False),
    "dtu_tf32_deterministic": ("dtu", 640, 512, 1, "tf32", 1, False, True),
}
WORST = {}


@pytest.fixture(autouse=True)
def _grad_mode():
    with torch.enable_grad():            # conftest runs GPU tests under no_grad by default
        yield


def _is_tf32(t):
    return bool((t.contiguous().view(torch.int32) & 0x1FFF).eq(0).all())


def _sample(B, W, H, seed, V=3):
    imgs, pm, dmin, dint = synth.make_inputs(B=B, V=V, W=W, H=H, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    depths, masks = {}, {}
    for l in range(3):
        hl, wl = H >> l, W >> l
        depths[f"level_{l}"] = (dmin + 100.0 + 40.0 * torch.rand(B, hl, wl, generator=g)).to(DEV)
        masks[f"level_{l}"] = (torch.rand(B, hl, wl, generator=g) > 0.2).to(DEV)
    return {"imgs": imgs.to(DEV), "proj_mats": pm.to(DEV),
            "init_depth_min": torch.full((B, 1), dmin, device=DEV),
            "depth_interval": torch.full((B, 1), dint, device=DEV), "depths": depths, "masks": masks}


# ------------------------------------------------------------------------------- recording
class Recorder:
    def __init__(self):
        self.on = True
        self.conv, self.conv_bwd = [], []
        self.warp, self.warp_bwd = [], []
        self.reg, self.reg_bwd = [], []


def _wrap(monkeypatch, fn_cls, record_fwd, record_bwd, rec, calls, bwd_calls):
    fwd0, bwd0 = fn_cls.forward, fn_cls.backward

    def forward(ctx, *args):
        if not rec.on:
            ctx.rec_id = None
            return fwd0(ctx, *args)
        ctx.rec_id = len(calls)
        f0 = _lib.fallback_count()
        out = fwd0(ctx, *args)
        calls.append(record_fwd(args, out, _lib.fallback_count() - f0))
        return out

    def backward(ctx, *grads):
        f0 = _lib.fallback_count()
        out = bwd0(ctx, *grads)
        if ctx.rec_id is not None:
            bwd_calls.append(dict(id=ctx.rec_id, fb=_lib.fallback_count() - f0,
                                  **record_bwd(grads, out)))
        return out

    # keep the originals' signatures: autograd.Function binds default arguments by them
    forward.__signature__ = inspect.signature(fwd0)
    monkeypatch.setattr(fn_cls, "forward", staticmethod(forward))
    monkeypatch.setattr(fn_cls, "backward", staticmethod(backward))


@pytest.fixture
def rec(monkeypatch):
    r = Recorder()
    vol = ops.volume_storage

    def conv_fwd(args, y, fb):
        x, w, kind, stride, precision = args
        return dict(x=vol(x.detach()).clone(), w=w.detach().clone(), kind=kind, stride=stride,
                    precision=precision, y=vol(y).clone(), fb=fb)

    def conv_bwd(grads, out):
        gx, gw = out[:2]
        return dict(gy=vol(grads[0]).clone(), gx=None if gx is None else vol(gx).clone(),
                    gw=None if gw is None else gw.clone())

    def warp_fwd(args, cost, fb):
        feats, proj, dv, G = args
        f = feats.detach().permute(0, 1, 3, 4, 2).clone(memory_format=torch.contiguous_format)
        return dict(f=f, P=proj.clone(), dv=dv.clone(), G=G, cost=vol(cost).clone())

    def warp_bwd(grads, out):
        return dict(gcost=vol(grads[0]).clone(), gf=out[0].permute(0, 1, 3, 4, 2).clone())

    def reg_fwd(args, out, fb):
        logits, dv = args
        return dict(logits=logits.detach().contiguous().clone(), dv=dv.clone(),
                    depth=out[0].detach().clone(), conf=out[1].clone())

    def reg_bwd(grads, out):
        return dict(gdepth=grads[0].contiguous().clone(), glogits=out[0].clone())

    _wrap(monkeypatch, AG.Conv3dFn, conv_fwd, conv_bwd, r, r.conv, r.conv_bwd)
    _wrap(monkeypatch, AG.WarpCostFn, warp_fwd, warp_bwd, r, r.warp, r.warp_bwd)
    _wrap(monkeypatch, AG.RegressFn, reg_fwd, reg_bwd, r, r.reg, r.reg_bwd)
    return r


@pytest.fixture
def det_switch():
    state = {"on": False}
    yield state
    if state["on"]:
        torch.use_deterministic_algorithms(False)


# ------------------------------------------------------------------------------- checks
def _note(kernel, need, bias=None):
    w = WORST.setdefault(kernel, [0.0, 0.0])
    w[0] = max(w[0], need)
    if bias is not None:
        w[1] = max(w[1], abs(bias))


def conv_report(got, want, A, kernel, r, r_op):
    """The checks of one convolution output (forward or data gradient) -> (bound ok, bias ok,
    worst voxel of R.bound_excess, eps needed beyond r_op, operand bias or None)."""
    ok, worst = R.bound_excess(got, want, A, EPS[kernel] + r_op, r)
    need = max(0.0, worst["eps_needed"] - r_op)
    bias = R.operand_bias(got, want) if r_op else None
    return ok, bias is None or abs(bias) <= BIAS_MAX, worst, need, bias


def _check_conv(tag, kernel, got, want, A, r, r_op):
    ok, bias_ok, worst, need, bias = conv_report(got, want, A, kernel, r, r_op)
    _note(kernel, need, bias)
    bias_txt = "" if bias is None else f", operand bias {bias:+.2e}"
    print(f"[train-fp64] {tag} [{kernel}]: eps needed {need:.3e} (eps {EPS[kernel]:.3e}"
          f"{' + r_op' if r_op else ''}){bias_txt}")
    assert ok, (f"{tag} [{kernel}]: |y - y64| exceeds eps*A + r_op*A + r|y64| + tiny; worst voxel "
                f"(b,d,h,w,c)={worst['at']} h%16={worst['h16']} w%8={worst['w8']}: got "
                f"{worst['got']!r}, float64 {worst['want']!r}, A={worst['A']:.4e}, needs eps "
                f"{need:.3e} > {EPS[kernel]:.3e} (r_op {r_op:.3e}, r {r:.3e})")
    assert bias_ok, (
        f"{tag} [{kernel}]: operand bias {bias:+.3e} exceeds {BIAS_MAX:.3e}: the tensor-core "
        f"operand was not rounded to nearest")


def _tc_kernel(kind, stride):
    return "tma" if kind == ops.CONV and stride == 1 else "tma2"


def _check_conv_calls(case, rec, tf32):
    assert len(rec.conv) == 33, f"{case}: {len(rec.conv)} forward calls, want 33"
    bwd = {b["id"]: b for b in rec.conv_bwd}
    assert len(rec.conv_bwd) == 33 and sorted(bwd) == list(range(33)), \
        f"{case}: backward calls for forward ids {sorted(bwd)}"
    fallbacks = set()
    for i, c in enumerate(rec.conv):
        level, name = LEVELS[i // 11], LAYERS[i % 11]
        tag = f"{case} L{level} {name}"
        kind, stride = c["kind"], c["stride"]
        assert (kind, stride) == KINDS[name], f"{tag}: kind {kind} stride {stride}"
        assert c["precision"] == (ops.TF32 if tf32 else ops.FP32), tag
        x, wt, y = c["x"], c["w"], c["y"]
        b = bwd[i]
        # ---- forward
        if c["fb"]:
            fallbacks.add((level, name, "forward"))
        tc = tf32 and not c["fb"]
        w64 = R.pack_weight(R.tf32_rna(wt) if tc else wt, kind)
        cout = w64.shape[-1]
        r = R.R_TF32 if tf32 and cout > 1 else 0.0
        r_op = R_OP if tc and not _is_tf32(x) else 0.0
        y64 = R.conv3d_ref(x, w64, kind, stride)
        A = R.magnitude(x, w64, kind, stride)
        _check_conv(f"{tag} forward {tuple(x.shape)}", _tc_kernel(kind, stride) if tc else "direct",
                    y, y64, A, r, r_op)
        del y64, A
        # ---- data gradient
        gy, gx = b["gy"], b["gx"]
        assert gx is not None and b["gw"] is not None, f"{tag}: no gradient"
        if b["fb"]:
            fallbacks.add((level, name, "dgrad"))
        tcb = tf32 and not b["fb"]
        wb64 = R.pack_weight(R.tf32_rna(wt) if tcb else wt, kind)
        cin = wb64.shape[-2]
        rb = R.R_TF32 if tf32 and cin > 1 else 0.0
        rb_op = R_OP if tcb and not _is_tf32(gy) else 0.0
        g64 = R.dgrad_ref(gy, wb64, kind, stride, x.shape[1:4])
        Ag = R.dgrad_ref(gy.abs(), wb64.abs(), kind, stride, x.shape[1:4])
        _check_conv(f"{tag} dgrad {tuple(gy.shape)}", _tc_kernel(kind, stride) if tcb else "direct",
                    gx, g64, Ag, rb, rb_op)
        del g64, Ag
        # ---- weight gradient, of the operand the forward kernel read
        xop = R.tf32_rna(x) if tc else x
        dw = R.pack_weight(b["gw"], kind)
        want = WG.wgrad_ref(xop, gy, kind, stride)
        Aw = WG.wgrad_magnitude(xop, gy, kind, stride)
        ok, worst = WG.wgrad_bound_excess(dw, want, Aw, EPS_WGRAD)
        _note("wgrad", worst["eps_needed"])
        print(f"[train-fp64] {tag} wgrad: eps needed {worst['eps_needed']:.3e} "
              f"(eps {EPS_WGRAD:.3e})")
        assert ok, (f"{tag} wgrad: worst (tap, cin, cout)={worst['at']}: got {worst['got']!r}, "
                    f"float64 {worst['want']!r}, A={worst['A']:.4e}, needs eps "
                    f"{worst['eps_needed']:.3e} > {EPS_WGRAD:.3e}")
        del want, Aw
    return fallbacks


def _check_k1_k3(case, rec):
    assert len(rec.warp) == len(rec.warp_bwd) == len(rec.reg) == len(rec.reg_bwd) == 3, case
    wb = {b["id"]: b for b in rec.warp_bwd}
    rb = {b["id"]: b for b in rec.reg_bwd}
    for i, c in enumerate(rec.warp):
        tag = f"{case} L{LEVELS[i]}"
        B, V, h, w, C = c["f"].shape
        fam = "staged" if ops.ladder_supported(V, C, c["G"]) else "gather"
        rep = W.check_cost(c["cost"], c["f"], c["P"], c["dv"], c["G"], EPS_K1[fam])
        print(f"[train-fp64] {tag} warp_cost [{fam}]: {rep.describe()}")
        assert rep.ok, f"{tag} warp_cost [{fam}]: {rep.describe()}"
        b = wb[i]
        rep = W.check_warp_cost_bwd(b["gf"], c["f"], c["P"], c["dv"], b["gcost"], c["G"],
                                    EPS_K1["bwd"])
        print(f"[train-fp64] {tag} warp_cost_bwd: {rep.describe()}")
        assert rep.ok, f"{tag} warp_cost_bwd: {rep.describe()}"
    for i, c in enumerate(rec.reg):
        tag = f"{case} L{LEVELS[i]}"
        # the index the kernel used for the confidence window: the same kernel, asked for it
        depth, conf, index, _ = ops.regress(c["logits"], c["dv"], want_index=True)
        assert torch.equal(depth, c["depth"]) and torch.equal(conf, c["conf"]), tag
        reps = RG.check_regress(c["logits"], c["dv"], c["depth"], c["conf"], index,
                                eps=EPS_K3["k3"])
        for k in ("depth", "conf"):
            print(f"[train-fp64] {tag} regress {k}: {reps[k].describe()}")
            assert reps[k].ok, f"{tag} regress {k}: {reps[k].describe()}"
        wrong, amb, first = reps["index"]
        assert wrong == 0, f"{tag}: {wrong} wrong indices, first at (b, y, x) = {first}"
        b = rb[i]
        g64, b0, A = RG.regress_bwd_ref(c["logits"], c["dv"], b["gdepth"])
        rep = RG.check(b["glogits"], g64, b0, A, EPS_K3["k3_bwd"], ("b", "d", "y", "x"))
        print(f"[train-fp64] {tag} regress_bwd: {rep.describe()}")
        assert rep.ok, f"{tag} regress_bwd: {rep.describe()}"


def _expected_fallbacks(tf32, G):
    if not tf32:
        return set()
    fb = {(l, "prob", "dgrad") for l in LEVELS}          # Cout = 1: a 4 -> 8 adjoint
    if G == 1:
        fb.add((1, "conv0", "dgrad"))                      # 8 -> 16: no stride-1 kernel
    if G in (2, 4):                                        # 4 -> 8 (G = 2 zero-padded to 4)
        fb |= {(l, "conv0", "forward") for l in LEVELS}
    return fb


@pytest.mark.parametrize("case", list(CASES))
def test_training_step_vs_fp64(case, rec, det_switch):
    data, W_, H, B, precision, G, update, det = CASES[case]
    tf32 = precision == "tf32"
    if det:
        os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
        torch.use_deterministic_algorithms(True)
        det_switch["on"] = True
    a = train.build_parser().parse_args(["--precision", precision, "--optimizer", "sgd",
                                         "--num_groups", str(G)])
    torch.manual_seed(0)
    model = train.build_model(a, DEV)
    tr = train.Trainer(a, model, DEV)
    if update:
        # every recorded call then runs after a weight change: a stale operand image of the
        # previous weights would show
        rec.on = False
        tr.train_step(_sample(B, W_, H, seed=100))
        rec.on = True
    f0 = _lib.fallback_count()
    loss, _ = tr.train_step(_sample(B, W_, H, seed=B))
    torch.cuda.synchronize()
    n_fb = _lib.fallback_count() - f0
    assert torch.isfinite(loss).item()
    print(f"[train-fp64] {case}: {data} {W_}x{H} B={B} {precision} G={G}: loss {loss.item():.5f}")
    with torch.no_grad():
        fallbacks = _check_conv_calls(case, rec, tf32)
        want = _expected_fallbacks(tf32, G)
        assert fallbacks == want, f"{case}: fallback layers {sorted(fallbacks)}, want {sorted(want)}"
        assert n_fb == len(want), f"{case}: {n_fb} fallback launches in the step, want {len(want)}"
        _check_k1_k3(case, rec)
    print(f"[train-fp64] worst so far (eps needed beyond r_op, |bias|): "
          + ", ".join(f"{k} {v[0]:.2e} / {v[1]:.2e}" for k, v in sorted(WORST.items())))
