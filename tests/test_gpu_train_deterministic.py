"""Bit-reproducible training on the GPU (torch.use_deterministic_algorithms(True)):

  * per kernel, at the training shapes: casmvs_warp_cost_bwd_det at the three cascade levels
    (variance and G = 8, B = 1 / 2, V = 3 / 5) and casmvs_conv3d_wgrad_det at every CostRegNet
    layer of the three levels are within the float64 bounds (warp_cost_fp64.check_warp_cost_bwd,
    conv3d_wgrad_fp64.wgrad_bound_excess), the atomic kernels are within the same bounds, and two
    calls on freshly allocated, differently offset buffers are torch.equal;
    casmvs_upsample2x_bilinear_bwd at FeatureNet's two upsamples against torch's float64 CPU
    backward, in both layouts;
  * whole training steps (DTU 640x512 and BlendedMVS 768x576, B = 1 / 2, fp32 / tf32) run under
    deterministic algorithms, and two steps from deep-copied states are torch.equal in the loss,
    the metric sums, every gradient, parameter and buffer;
  * two `train.main(..., --deterministic, --seed 0)` processes of two epochs write byte-identical
    metrics.jsonl files and torch.equal checkpoints."""
import copy
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from casmvsnet_pl_b200 import _lib, ops, synth, train            # noqa: E402
from oracle import conv3d_fp64 as K                                # noqa: E402
from oracle import conv3d_wgrad_fp64 as WG                         # noqa: E402
from oracle import warp_cost_fp64 as W                             # noqa: E402

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS_K1 = 2.0 ** -22          # the fp64 tolerance of casmvs_warp_cost_bwd (test_gpu_warp_cost_fp64)
LOOSE_K1 = 2.0 ** -4
# weight gradient: eps per magnitude sum |x| |gy|, the largest power of two within 4x of the
# worst need over this file's layers (5.2e-8, deterministic and atomic kernels alike) on an
# H100 80GB HBM3 at a 400 W power limit; the need is printed per layer
EPS_WGRAD = 2.0 ** -23
# upsample: the same float32 weights as ATen, summed in another order: <= 16 roundings of sum |w g|
EPS_UP = 2.0 ** -20


@pytest.fixture(autouse=True)
def _grad_mode():
    with torch.enable_grad():            # conftest runs GPU tests under no_grad by default
        yield


@pytest.fixture
def det():
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(False)


def _offset_copy(t, offset):
    """A copy of t in a fresh allocation, `offset` floats (a multiple of 4) into it."""
    buf = torch.empty(t.numel() + offset, device=t.device, dtype=t.dtype)
    out = buf[offset:].view(t.shape)
    out.copy_(t)
    return out


# ------------------------------------------------------------------------------- K1 backward
_LEVELS = {0: (8, 8), 1: (16, 32), 2: (32, 48)}              # level: C, D at 640x512
K1 = {f"L{l}_g{G}_b{B}_v{V}": (B, V, C, G, 512 >> l, 640 >> l, D, l)
      for l, (C, D) in _LEVELS.items() for G in (1, 8) for B, V in ((1, 3), (2, 5))}


def _k1_inputs(name):
    B, V, C, G, h, w, D, l = K1[name]
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, name)))
    f = torch.randn(B, V, h, w, C, generator=g, device=DEV)
    P = synth.projection_matrices(V, w << l, h << l)[:, l].unsqueeze(0).repeat(B, 1, 1, 1)
    P[:, :, 0, 2] += torch.arange(B).view(B, 1) * 1.37
    P = P.to(DEV).contiguous()
    step = synth.DEPTH_INTERVAL * (1 << l)
    first = 600.0 - D / 2 * step + 25.0 * torch.rand(B, 1, h, w, generator=g, device=DEV)
    dv = (first + step * torch.arange(D, device=DEV).view(1, D, 1, 1)).contiguous()
    gcost = torch.randn(B, D, h, w, C if G == 1 else G, generator=g, device=DEV)
    return f, P, dv, gcost


def _k1_det(spec, f, P, dv, gcost, offset):
    B, V, C, G, h, w, D, _ = spec
    lib = _lib.load()
    f, P, dv, gcost = (_offset_copy(t, offset) for t in (f, P, dv, gcost))
    gf = _offset_copy(torch.full_like(f, float("nan")), offset)
    nbytes = lib.casmvs_warp_cost_bwd_det_workspace_bytes(B, V, C, D, h, w)
    ws = torch.empty(nbytes + 256 * (offset + 1), dtype=torch.uint8, device=DEV)
    wp = ws[256 * offset:]
    _lib.check(lib.casmvs_warp_cost_bwd_det(ops._ptr(f), ops._ptr(P), ops._ptr(dv), ops._ptr(gcost),
                                            ops._ptr(gf), B, V, C, D, h, w, G, ops._ptr(wp), wp.numel(),
                                            ops._stream()), "warp_cost_bwd_det")
    return gf.clone(), nbytes


def _k1_atomic(spec, f, P, dv, gcost):
    B, V, C, G, h, w, D, _ = spec
    gf = torch.zeros_like(f)
    _lib.check(_lib.load().casmvs_warp_cost_bwd(ops._ptr(f), ops._ptr(P), ops._ptr(dv), ops._ptr(gcost),
                                                ops._ptr(gf), B, V, C, D, h, w, G, ops._stream()),
               "warp_cost_bwd")
    return gf


@pytest.mark.parametrize("name", list(K1))
def test_warp_cost_bwd_det(name):
    spec = K1[name]
    f, P, dv, gcost = _k1_inputs(name)
    a, nbytes = _k1_det(spec, f, P, dv, gcost, 0)
    b, _ = _k1_det(spec, f, P, dv, gcost, 12)
    assert torch.equal(a, b), f"{name}: two calls differ"
    rep = W.check_warp_cost_bwd(a, f, P, dv, gcost, spec[3], EPS_K1)
    print(f"[det] {name}: workspace {nbytes / 1e9:.3f} GB; {rep.describe()}")
    assert rep.ok, f"{name}: {rep.describe()}"
    assert rep.loose_share <= LOOSE_K1, f"{name} loose: {rep.describe()}"
    at = _k1_atomic(spec, f, P, dv, gcost)
    rep_at = W.check_warp_cost_bwd(at, f, P, dv, gcost, spec[3], EPS_K1)
    print(f"[det] {name}: atomic kernel: {rep_at.describe()}; max |det - atomic| "
          f"{(a - at).abs().max().item():.3e}")
    assert rep_at.ok, f"{name} atomic: {rep_at.describe()}"


# ------------------------------------------------------------------------------- weight gradient
# CostRegNet layers: (name, kind, stride, Cin, Cout, scale of the layer input's dims)
_LAYERS = [("conv0", K.CONV, 1, None, 8, 1), ("conv1", K.CONV, 2, 8, 16, 1), ("conv2", K.CONV, 1, 16, 16, 2),
           ("conv3", K.CONV, 2, 16, 32, 2), ("conv4", K.CONV, 1, 32, 32, 4), ("conv5", K.CONV, 2, 32, 64, 4),
           ("conv6", K.CONV, 1, 64, 64, 8), ("conv7", K.CONV_TRANSPOSE, 2, 64, 32, 8),
           ("conv9", K.CONV_TRANSPOSE, 2, 32, 16, 4), ("conv11", K.CONV_TRANSPOSE, 2, 16, 8, 2),
           ("prob", K.CONV, 1, 8, 1, 1)]
WGRAD = {}
for _l, (_C, _D) in _LEVELS.items():
    for _B in ((1, 2) if _l == 2 else (1,)):
        for _n, _kind, _s, _cin, _cout, _sc in _LAYERS:
            WGRAD[f"L{_l}_b{_B}_{_n}"] = (_B, _kind, _s, _cin or _C, _cout, _D // _sc, (512 >> _l) // _sc,
                                         (640 >> _l) // _sc)


def _wgrad_call(x, gy, B, ca, cb, xdims, ydims, stride, det, offset=0):
    lib = _lib.load()
    if not det:
        dw = torch.zeros(27, ca, cb, device=DEV)
        _lib.check(lib.casmvs_conv3d_wgrad(ops._ptr(x), ops._ptr(gy), ops._ptr(dw), B, ca, cb, *xdims,
                                           *ydims, stride, ops._stream()), "conv3d_wgrad")
        return dw
    x, gy = _offset_copy(x, offset), _offset_copy(gy, offset)
    dw = _offset_copy(torch.full((27, ca, cb), float("nan"), device=DEV), offset)
    nbytes = lib.casmvs_conv3d_wgrad_det_workspace_bytes(B, ca, cb, *ydims)
    ws = torch.empty(nbytes + 4 * offset, dtype=torch.uint8, device=DEV)[4 * offset:]
    _lib.check(lib.casmvs_conv3d_wgrad_det(ops._ptr(x), ops._ptr(gy), ops._ptr(dw), B, ca, cb, *xdims,
                                           *ydims, stride, ops._ptr(ws), ws.numel(), ops._stream()),
               "conv3d_wgrad_det")
    return dw.clone()


@pytest.mark.parametrize("name", list(WGRAD))
def test_conv3d_wgrad_det(name):
    B, kind, stride, cin, cout, D, h, w = WGRAD[name]
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, name)))
    x = torch.randn(B, D, h, w, cin, generator=g, device=DEV)
    Do, ho, wo = K.out_dims(kind, stride, D, h, w)
    gy = torch.randn(B, Do, ho, wo, cout, generator=g, device=DEV)
    if kind == K.CONV:
        args = (x, gy, B, cin, cout, (D, h, w), (Do, ho, wo), stride)
        want, A = WG.wgrad_ref(x, gy, kind, stride), WG.wgrad_magnitude(x, gy, kind, stride)
    else:                                    # the library's roles: gy strided, (27, Cout, Cin)
        args = (gy, x, B, cout, cin, (Do, ho, wo), (D, h, w), 2)
        want = WG.wgrad_ref(x, gy, kind).transpose(1, 2).contiguous()
        A = WG.wgrad_magnitude(x, gy, kind).transpose(1, 2).contiguous()
    a = _wgrad_call(*args, det=True)
    b = _wgrad_call(*args, det=True, offset=36)
    assert torch.equal(a, b), f"{name}: two calls differ"
    ok, worst = WG.wgrad_bound_excess(a, want, A, EPS_WGRAD)
    at = _wgrad_call(*args, det=False)
    ok_at, worst_at = WG.wgrad_bound_excess(at, want, A, EPS_WGRAD)
    print(f"[det] wgrad {name}: eps needed {worst['eps_needed']:.2e} (atomic kernel "
          f"{worst_at['eps_needed']:.2e})")
    assert ok, f"{name}: {worst}"
    assert ok_at, f"{name} atomic: {worst_at}"


# ------------------------------------------------------------------------------- upsample
@pytest.mark.parametrize("N,h,w", [(3, 128, 160), (3, 256, 320), (6, 144, 192), (2, 1, 3), (1, 5, 2)])
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_upsample2x_bwd_vs_torch_fp64(N, h, w, layout):
    from casmvsnet_pl_b200 import autograd as AG
    g = torch.Generator().manual_seed(N * h + w)
    x = torch.randn(N, 32, h, w, generator=g)
    gy = torch.randn(N, 32, 2 * h, 2 * w, generator=g)
    x64 = x.double().requires_grad_(True)
    F.interpolate(x64, scale_factor=2, mode="bilinear", align_corners=True).backward(gy.double())
    up = torch.ones_like(x64, requires_grad=True)
    F.interpolate(up, scale_factor=2, mode="bilinear", align_corners=True).backward(gy.double().abs())
    A = up.grad                                       # sum |w g| over each input's contributions
    fmt = torch.channels_last if layout == "nhwc" else torch.contiguous_format
    outs = []
    for offset in (0, 8):
        xd = x.to(DEV).contiguous(memory_format=fmt).requires_grad_(True)
        gyd = _offset_copy(gy.to(DEV).contiguous(memory_format=fmt), offset) if layout == "nchw" else \
            gy.to(DEV).contiguous(memory_format=fmt)
        y = AG.Upsample2xFn.apply(xd)
        assert torch.equal(y, F.interpolate(xd.detach(), scale_factor=2, mode="bilinear", align_corners=True))
        y.backward(gyd)
        assert xd.grad.is_contiguous(memory_format=fmt)
        outs.append(xd.grad.cpu())
    assert torch.equal(outs[0], outs[1])
    # torch's CUDA backward: the same float32 weights and products, added by atomics
    xt = x.to(DEV).contiguous(memory_format=fmt).requires_grad_(True)
    F.interpolate(xt, scale_factor=2, mode="bilinear", align_corners=True).backward(
        gy.to(DEV).contiguous(memory_format=fmt))
    d_torch = (outs[0].double() - xt.grad.cpu().double()).abs()
    assert (d_torch <= EPS_UP * A).all(), (d_torch - EPS_UP * A).max().item()
    # float64: besides the sums, ATen's float32 source coordinate scale * o (<= max(h, w)) rounds
    # each lambda by up to 2^-23 max(h, w), and each of the <= 16 terms has |g| <= max |gy|
    d64 = (outs[0].double() - x64.grad).abs()
    slack = EPS_UP * A + 2.0 ** -22 * max(h, w) * 16 * gy.abs().max().item()
    print(f"[det] upsample {N}x32x{h}x{w} {layout}: max |err| vs float64 {d64.max():.2e} "
          f"(slack {slack.min():.2e}..{slack.max():.2e}), vs torch CUDA {d_torch.max():.2e}")
    assert (d64 <= slack).all(), (d64 - slack).max().item()


def test_upsample2x_routes_by_the_switch(det):
    from casmvsnet_pl_b200 import autograd as AG
    x = torch.randn(2, 32, 8, 10, device=DEV, requires_grad=True)
    AG.upsample2x(x).sum().backward()                 # ATen's backward would raise here
    torch.use_deterministic_algorithms(False)
    y = AG.upsample2x(x)
    assert y.grad_fn.name() != "Upsample2xFnBackward"


# ------------------------------------------------------------------------------- whole steps
def _sample(B, W, H, seed):
    imgs, pm, dmin, dint = synth.make_inputs(B=B, V=3, W=W, H=H, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    depths, masks = {}, {}
    for l in range(3):
        hl, wl = H >> l, W >> l
        depths[f"level_{l}"] = (dmin + 100.0 + 40.0 * torch.rand(B, hl, wl, generator=g)).to(DEV)
        masks[f"level_{l}"] = (torch.rand(B, hl, wl, generator=g) > 0.2).to(DEV)
    return {"imgs": imgs.to(DEV), "proj_mats": pm.to(DEV),
            "init_depth_min": torch.full((B, 1), dmin, device=DEV),
            "depth_interval": torch.full((B, 1), dint, device=DEV), "depths": depths, "masks": masks}


def _step(model, a, s):
    tr = train.Trainer(a, model, DEV)
    loss, metrics = tr.train_step(s)
    return loss, metrics


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("data,W,H", [("dtu", 640, 512), ("blendedmvs", 768, 576)])
def test_training_step_is_bit_reproducible(det, data, W, H, B, precision):
    a = train.build_parser().parse_args(["--precision", precision, "--optimizer", "sgd"])
    torch.manual_seed(0)
    model = train.build_model(a, DEV)
    twin = copy.deepcopy(model)
    s = _sample(B, W, H, seed=B)
    torch.cuda.reset_peak_memory_stats()
    l1, m1 = _step(model, a, s)
    peak = torch.cuda.max_memory_allocated() / 1e9
    l2, m2 = _step(twin, a, s)
    print(f"[det] {data} {W}x{H} B={B} {precision}: loss {l1.item():.6f}, peak allocated {peak:.2f} GB")
    assert torch.isfinite(l1).item()
    assert torch.equal(l1, l2) and torch.equal(m1, m2)
    for (k, p), q in zip(model.named_parameters(), twin.parameters()):
        assert p.grad is not None, k
        assert torch.equal(p.grad, q.grad), f"gradient of {k}"
        assert torch.equal(p, q), k
    for (k, u), v in zip(model.named_buffers(), twin.buffers()):
        assert torch.equal(u, v), k


# ------------------------------------------------------------------------------- processes
@pytest.fixture(scope="module")
def dtu_root(tmp_path_factory):
    from casmvsnet_pl_b200.synth_scenes import make_dtu_train
    return make_dtu_train(str(tmp_path_factory.mktemp("dtu_det")), seed=0)


def test_two_processes_write_the_same_run(dtu_root, tmp_path):
    argv = ["--root_dir", dtu_root, "--train_list", os.path.join(dtu_root, "lists", "train.txt"),
            "--val_list", os.path.join(dtu_root, "lists", "val.txt"), "--num_epochs", "2",
            "--optimizer", "adam", "--log_every", "1", "--num_workers", "2", "--exp_name", "det",
            "--deterministic", "--seed", "0"]
    code = "import sys\nsys.path.insert(0, %r)\nfrom casmvsnet_pl_b200 import train\ntrain.main(sys.argv[1:])\n" % ROOT
    runs = []
    for i in range(2):
        cwd = tmp_path / f"run{i}"
        cwd.mkdir()
        subprocess.run([sys.executable, "-c", code] + argv, check=True, cwd=str(cwd), timeout=900)
        runs.append(cwd)
    logs = [open(r / "logs" / "det" / "metrics.jsonl", "rb").read() for r in runs]
    assert logs[0] and logs[0] == logs[1]
    names = sorted(os.listdir(runs[0] / "ckpts" / "det"))
    assert names and names == sorted(os.listdir(runs[1] / "ckpts" / "det"))
    for n in names:
        c0, c1 = (torch.load(r / "ckpts" / "det" / n, map_location="cpu") for r in runs)
        assert c0["epoch"] == c1["epoch"] and c0["global_step"] == c1["global_step"]
        assert c0["state_dict"].keys() == c1["state_dict"].keys()
        for k, v in c0["state_dict"].items():
            assert torch.equal(v, c1["state_dict"][k]), f"{n}: {k}"
    lines = logs[0].count(b"\n")
    print(f"[det] two processes: {lines} log lines, checkpoints {names} identical")
