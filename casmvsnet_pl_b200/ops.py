"""torch-tensor wrappers over the C ABI (include/casmvs.h).

PyTorch is plumbing here: it owns device memory and the stream; every op below
is a call into libcasmvs.so.  CPU tensors are rejected — there is no fallback
(SURVEY.md §8b: `eval.py --cpu` stays an oracle-only mode).
"""
from __future__ import annotations

import ctypes
import functools
import math

import torch

from . import _lib
from ._lib import (BLOCKED, CONV, CONV_PLANAR, CONV_TRANSPOSE, FP32, FUSED_TAIL, INVERSE_DEPTH, KEEP_FP32_OUT, NCHW,  # noqa: F401
                   NHWC, PRECISIONS, TF32, check)

_checked_devices = set()


def _stream():
    """The current stream of the CURRENT device; every op runs under `_on_tensor_device`, which
    makes the tensors' device current first (the reference allows `model.to("cuda:1")` while
    cuda:0 is current)."""
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _on_tensor_device(fn):
    """Run `fn` with the device of its first CUDA tensor argument (or `device=` keyword) current:
    kernel launches, cudaFuncSetAttribute, the SM count and the library's cudaMalloc'ed
    operand images are all per-device state."""
    @functools.wraps(fn)
    def wrapper(*args, **kw):
        dev = kw.get("device")
        if dev is None:
            dev = next((a.device for a in args if torch.is_tensor(a) and a.is_cuda), None)
        else:
            dev = torch.device(dev)
        if dev is None or dev.type != "cuda" or dev.index is None or \
                dev.index == torch.cuda.current_device():
            return fn(*args, **kw)
        with torch.cuda.device(dev):
            return fn(*args, **kw)
    return wrapper


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _require_cuda(*tensors):
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise _lib.CasMVSError(
                "casmvsnet_pl_b200 ops need CUDA tensors on a H100 (no CPU fallback); "
                f"got a tensor on {t.device}")
        if t.dtype != torch.float32:
            raise _lib.CasMVSError(f"fp32 only (reference opt.py:69-70), got {t.dtype}")
    first = next((t for t in tensors if t is not None), None)
    if first is None:
        return
    for t in tensors:
        if t is not None and t.device != first.device:
            raise _lib.CasMVSError(f"tensors on different devices: {first.device} and {t.device}")
    dev = first.device.index
    if dev is None:
        dev = torch.cuda.current_device()
    if dev not in _checked_devices:
        check(_lib.load().casmvs_device_check(dev), "device_check")
        _checked_devices.add(dev)


def _no_grad_only(*tensors):
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors):
        raise _lib.CasMVSError(
            "the H100 engine is forward-only this round (SURVEY.md §8f-1): call it under "
            "torch.no_grad() or with tensors that do not require grad")


def is_channels_last_feats(feats):
    """feats (..., C, h, w): True if physically (..., h, w, C) dense."""
    C, h, w = feats.shape[-3:]
    st = feats.stride()
    if not (st[-3] == 1 and st[-1] == C and st[-2] == w * C):
        return False
    expect = h * w * C
    for size, s in zip(reversed(feats.shape[:-3]), reversed(st[:-3])):
        if size != 1 and s != expect:
            return False
        expect *= size
    return True


def as_volume_view(buf_ndhwc):
    """(B,D,h,w,C) buffer -> logical (B,C,D,h,w) view (channels_last_3d strides)."""
    return buf_ndhwc.permute(0, 4, 1, 2, 3)


def volume_storage(x):
    """logical (B,C,D,h,w) -> dense (B,D,h,w,C) storage (copy only if needed)."""
    v = x.permute(0, 2, 3, 4, 1)
    return v if v.is_contiguous() else v.contiguous()


# --------------------------------------------------------------------------- K1
@_on_tensor_device
def warp_cost(feats, proj_mats, depth_values, num_groups=1, out_layout=NHWC, round_tf32=False):
    """Fused homography warp + variance / group-wise-correlation cost volume.

    feats (B,V,C,h,w) (any strides; channels-last storage is used as is),
    proj_mats (B,V-1,3,4), depth_values (B,D,h,w).
    Returns the LOGICAL (B,Cout,D,h,w) tensor; with out_layout=NHWC its memory
    is (B,D,h,w,Cout) (torch channels_last_3d), what the conv stack consumes.
    """
    _require_cuda(feats, proj_mats, depth_values)
    _no_grad_only(feats)
    B, V, C, h, w = feats.shape
    D = depth_values.shape[1]
    lib = _lib.load()
    if is_channels_last_feats(feats):
        flayout, fbuf = NHWC, feats
    else:
        flayout, fbuf = NCHW, feats.contiguous()
    proj = proj_mats.contiguous()
    dv = depth_values.contiguous()
    assert proj.shape == (B, V - 1, 3, 4) and dv.shape == (B, D, h, w)
    cout = C if num_groups == 1 else num_groups
    ws_bytes = lib.casmvs_warp_cost_workspace_bytes(flayout, B, V, C, h, w)
    ws = torch.empty(ws_bytes // 4, device=feats.device, dtype=torch.float32) if ws_bytes else None
    if out_layout == NHWC:
        out = torch.empty(B, D, h, w, cout, device=feats.device, dtype=torch.float32)
    else:
        out = torch.empty(B, cout, D, h, w, device=feats.device, dtype=torch.float32)
    check(lib.casmvs_warp_cost_fwd(_ptr(fbuf), flayout, _ptr(proj), _ptr(dv), _ptr(out),
                                   out_layout | (_lib.ROUND_TF32 if round_tf32 else 0),
                                   B, V, C, D, h, w, num_groups, _ptr(ws),
                                   ws_bytes, _stream()), "warp_cost")
    return as_volume_view(out) if out_layout == NHWC else out


@_on_tensor_device
def homo_warp(src_feat, proj_mat, depth_values):
    """models/modules.py:52-92.  src_feat (B,C,h,w), proj_mat (B,3,4),
    depth_values (B,D,h,w) -> (B,C,D,h,w) contiguous (reference layout)."""
    _require_cuda(src_feat, proj_mat, depth_values)
    _no_grad_only(src_feat)
    B, C, h, w = src_feat.shape
    D = depth_values.shape[1]
    lib = _lib.load()
    if is_channels_last_feats(src_feat):
        fbuf = src_feat
    else:
        fbuf = torch.empty(B, h, w, C, device=src_feat.device, dtype=torch.float32)
        check(lib.casmvs_nchw_to_nhwc(_ptr(src_feat.contiguous()), _ptr(fbuf), B, C, h * w,
                                      _stream()), "nchw_to_nhwc")
    out = torch.empty(B, C, D, h, w, device=src_feat.device, dtype=torch.float32)
    check(lib.casmvs_homo_warp_fwd(_ptr(fbuf), NHWC, _ptr(proj_mat.contiguous()),
                                   _ptr(depth_values.contiguous()), _ptr(out), NCHW,
                                   B, C, D, h, w, _stream()), "homo_warp")
    return out


# --------------------------------------------------------------------------- K2
def invalidate_weight_cache():
    """Drop ALL of the library's cached tensor-core operand images."""
    check(_lib.load().casmvs_invalidate_weight_cache(), "invalidate_weight_cache")


def release_weight_images(packed):
    """Drop the operand images keyed inside `packed`'s memory.  Called on every freshly
    allocated packed-weight buffer BEFORE it is filled: the caching allocator may hand out an
    address whose previous owner (an older packed buffer) still has images in the cache."""
    check(_lib.load().casmvs_release_weight_images(_ptr(packed), packed.numel() * packed.element_size()),
          "release_weight_images")


@_on_tensor_device
def pack_conv3d_weight(weight, kind):
    """torch Conv3d (Cout,Cin,3,3,3) / ConvTranspose3d (Cin,Cout,3,3,3) / Conv2d (Cout,Cin,3,3)
    [kind CONV_PLANAR: centre plane of a 1x3x3 kernel] -> [27][Cin][Cout]."""
    _require_cuda(weight)
    if kind == CONV_PLANAR:
        assert weight.dim() == 4 and tuple(weight.shape[2:]) == (3, 3)
    if kind in (CONV, CONV_PLANAR):
        cout, cin = weight.shape[:2]
    else:
        cin, cout = weight.shape[:2]
    out = torch.empty(27 * cin * cout, device=weight.device, dtype=torch.float32)
    release_weight_images(out)
    check(_lib.load().casmvs_pack_conv3d_weights(_ptr(weight.detach().contiguous()), kind, cin,
                                                 cout, _ptr(out), _stream()), "pack_conv3d")
    return out


@_on_tensor_device
def conv3d(x, w_packed, cin, cout, scale=None, shift=None, slope=1.0, skip=None,
           kind=CONV, stride=1, precision=FP32):
    """x logical (B,Cin,D,h,w) -> logical (B,Cout,Do,ho,wo); storage channels-last."""
    _require_cuda(x, w_packed, scale, shift, skip)
    _no_grad_only(x)
    xs = volume_storage(x)
    B, D, h, w, _ = xs.shape
    if kind == CONV_PLANAR:
        assert stride == 1
        Do, ho, wo = D, h, w
    elif kind == CONV:
        Do, ho, wo = (D - 1) // stride + 1, (h - 1) // stride + 1, (w - 1) // stride + 1
    else:
        Do, ho, wo = 2 * D, 2 * h, 2 * w
    y = torch.empty(B, Do, ho, wo, cout, device=x.device, dtype=torch.float32)
    sk = volume_storage(skip) if skip is not None else None
    check(_lib.load().casmvs_conv3d_fwd(_ptr(xs), _ptr(w_packed), _ptr(scale), _ptr(shift),
                                        float(slope), _ptr(sk), _ptr(y), B, cin, cout, D, h, w,
                                        kind, stride, precision, _stream()), "conv3d")
    return as_volume_view(y)


def conv3d_tensor_core(cin, cout, kind, stride, skip=False):
    """True when conv3d in the TF32 precision runs this layer on a tensor-core kernel, False
    when it falls back to the CUDA cores (casmvs_fallback_count)."""
    return bool(_lib.load().casmvs_conv3d_tensor_core(cin, cout, kind, stride, int(skip)))


def costreg_layer_info(cin, layer):
    lib = _lib.load()
    ci, co, kind, stride = (ctypes.c_int() for _ in range(4))
    wo, so, ho = (ctypes.c_size_t() for _ in range(3))
    check(lib.casmvs_costreg_layer_info(cin, layer, ci, co, kind, stride, wo, so, ho),
          "costreg_layer_info")
    return dict(cin=ci.value, cout=co.value, kind=kind.value, stride=stride.value,
                w_off=wo.value, scale_off=so.value, shift_off=ho.value)


def costreg_blocked_supported(cin, precision=TF32):
    """True when costreg runs blocked activations for this Cin and precision, and so accepts
    costreg(blocked=True) (the tensor-core kernels cover every layer)."""
    return bool(_lib.load().casmvs_costreg_blocked_supported(cin, precision))


@_on_tensor_device
def costreg(x, params, cin, precision=FP32, blocked=False, fused_tail=True):
    """Whole CostRegNet.  x logical (B,Cin,D,h,w) -> logits (B,D,h,w).  blocked=True (TF32
    only, where costreg_blocked_supported): x is a contiguous (B,Cin/4,D,h,w,4) tensor, e.g. from
    warp_cost_ladder(blocked=True).  The workspace is private, so by default conv11 and the prob
    head run as one kernel where the library has it (casmvs_costreg_tail_supported);
    fused_tail=False runs them as two layers (the same logits)."""
    _require_cuda(x, params)
    _no_grad_only(x)
    if blocked:
        if x.dim() != 6 or x.shape[-1] != 4 or x.shape[1] * 4 != cin or not x.is_contiguous():
            raise ValueError(f"costreg: blocked input must be a contiguous (B,{cin // 4},D,h,w,4) "
                             f"tensor, got {tuple(x.shape)}")
        xs = x
        B, _, D, h, w, _ = xs.shape
        precision |= BLOCKED
    else:
        xs = volume_storage(x)
        B, D, h, w, c = xs.shape
        assert c == cin
    if fused_tail:
        precision |= FUSED_TAIL
    lib = _lib.load()
    ws_bytes = lib.casmvs_costreg_workspace_bytes(B, cin, D, h, w)
    ws = torch.empty(ws_bytes // 4, device=x.device, dtype=torch.float32)
    logits = torch.empty(B, D, h, w, device=x.device, dtype=torch.float32)
    check(lib.casmvs_costreg_fwd(_ptr(xs), _ptr(params), _ptr(logits), B, cin, D, h, w,
                                 precision, _ptr(ws), ws_bytes, _stream()), "costreg")
    return logits


# --------------------------------------------------------------------------- K3
@_on_tensor_device
def regress(logits, depth_values, input_is_prob=False, want_index=False, want_prob=False,
            inverse=False, want_spread=False):
    """softmax + soft-argmax depth + confidence (+ index, prob).
    logits (B,D,h,w); depth_values (B,D,h,w) or (D,).  inverse=True regresses in 1/depth:
    depth = 1/sum_d p_d/depth_values_d (README "Wide depth ranges").  want_spread=True also
    returns the spread sqrt(sum_d p_d (depth_values_d - depth)^2) (B,h,w) as a fifth value
    (README "Adaptive depth ranges"); the other outputs are the same bits as without it."""
    if want_spread and inverse:
        raise _lib.CasMVSError("regress: want_spread is the adaptive mode's, not the inverse mode's")
    _require_cuda(logits, depth_values)
    _no_grad_only(logits)
    lg = logits.contiguous()
    B, D, h, w = lg.shape
    dv_vec = depth_values.dim() == 1
    dv = depth_values.contiguous()
    depth = torch.empty(B, h, w, device=lg.device, dtype=torch.float32)
    conf = torch.empty_like(depth)
    index = torch.empty(B, h, w, device=lg.device, dtype=torch.int64) if want_index else None
    prob = torch.empty_like(lg) if want_prob else None
    if want_spread:
        spread = torch.empty_like(depth)
        check(_lib.load().casmvs_regress_spread_fwd(_ptr(lg), _ptr(dv), int(dv_vec), int(bool(input_is_prob)),
                                                    _ptr(depth), _ptr(conf), _ptr(index), _ptr(prob),
                                                    _ptr(spread), B, D, h, w, _stream()), "regress")
        return depth, conf, index, prob, spread
    flags = int(bool(input_is_prob)) | (INVERSE_DEPTH if inverse else 0)
    check(_lib.load().casmvs_regress_fwd(_ptr(lg), _ptr(dv), int(dv_vec), flags,
                                         _ptr(depth), _ptr(conf), _ptr(index), _ptr(prob),
                                         B, D, h, w, _stream()), "regress")
    return depth, conf, index, prob


# --------------------------------------------------------------------------- K4
def _interval_args(depth_interval, B, device):
    """float -> (scalar, None); tensor (B,1)/(B,) -> (0.0, device (B,) tensor)."""
    if isinstance(depth_interval, (float, int)):
        return float(depth_interval), None
    t = depth_interval.reshape(-1).to(device=device, dtype=torch.float32).contiguous()
    if t.numel() == 1 and B > 1:
        t = t.expand(B).contiguous()
    assert t.numel() == B
    return 0.0, t


@_on_tensor_device
def depth_hypotheses(current_depth, n_depths, depth_interval, upsample=False):
    """get_depth_values (models/modules.py:34-49), optionally fused with the x2
    bilinear upsample of models/mvsnet.py:231-234.
    current_depth (B,1,h,w), or (B,h/2,w/2) when upsample=True -> (B,D,h,w)."""
    _require_cuda(current_depth)
    cur = current_depth.contiguous()
    if upsample:
        B, hi, wi = cur.shape
        h, w = 2 * hi, 2 * wi
    else:
        B, _, h, w = cur.shape
    step, step_dev = _interval_args(depth_interval, B, cur.device)
    # python-float interval: the reference forms n/2*interval in double, torch
    # then rounds the scalar to fp32 for the tensor op (modules.py:44)
    half = float(n_depths / 2 * step)
    out = torch.empty(B, n_depths, h, w, device=cur.device, dtype=torch.float32)
    check(_lib.load().casmvs_depth_hypotheses_fwd(_ptr(cur), int(upsample), half, step,
                                                  _ptr(step_dev), _ptr(out), B, n_depths, h, w,
                                                  _stream()), "depth_hypotheses")
    return out


def uniform_hypotheses(init_depth_min, depth_interval, n_depths, B, h, w, device):
    """models/mvsnet.py:213-229 -> (B,D,h,w)."""
    with torch.cuda.device(device):
        return _uniform_hypotheses(init_depth_min, depth_interval, n_depths, B, h, w, device)


def _uniform_hypotheses(init_depth_min, depth_interval, n_depths, B, h, w, device):
    dmin, dmin_dev = _interval_args(init_depth_min, B, device)
    step, step_dev = _interval_args(depth_interval, B, device)
    out = torch.empty(B, n_depths, h, w, device=device, dtype=torch.float32)
    check(_lib.load().casmvs_uniform_hypotheses_fwd(dmin, step, _ptr(dmin_dev), _ptr(step_dev),
                                                    _ptr(out), B, n_depths, h, w, _stream()),
          "uniform_hypotheses")
    return out


# --------------------------------------------------------------------------- inverse depth
class InverseSteps:
    """Rules 1-2 of the inverse-depth plane sweep (csrc/regress.cu, README "Wide depth ranges")
    for one forward: u_near = 1/near, u_far = 1/far and the per-stage plane spacing step[l] in
    1/depth, each a float (float depth parameters) or a (B,) float32 device tensor."""

    def __init__(self, u_near, u_far, step, B):
        self.u_near, self.u_far, self.step, self.B = u_near, u_far, step, B


def _depth_param(x, B):
    t = x.reshape(-1).to(torch.float32)
    return t.expand(B).contiguous() if t.numel() == 1 and B > 1 else t


def inverse_steps(init_depth_min, depth_interval, n_depths, interval_ratios, B, device=None):
    """u_near, u_far and s_l of the inverse-depth sweep (stage l = 0 finest .. len-1 coarsest).
    near = init_depth_min, far = the uniform mode's last coarse plane
    init_depth_min + (D-1)*depth_interval*ratio, formed in float32 as the hypothesis kernel forms
    it; then in float64, each rounded once to float32: u_near = 1/near, u_far = 1/far,
    s_top = (u_near - u_far)/(D_top - 1), s_l = s_top*ratio_l/ratio_top.
    Raises CasMVSError unless 0 < near < far, both finite.  Floats and CPU tensors are checked
    on the host; device tensors with one synchronise (skipped while a CUDA graph is captured:
    the capturing caller has run the same tensors eagerly first)."""
    top = len(n_depths) - 1
    D, r_top = n_depths[top], interval_ratios[top]
    if D < 2:
        raise _lib.CasMVSError("inverse depth sampling needs at least 2 planes in the coarsest stage")
    tensors = [t for t in (init_depth_min, depth_interval) if torch.is_tensor(t)]
    dev = tensors[0].device if tensors else torch.device("cpu")
    # the coarse stage's interval and far plane exactly as the uniform mode forms them
    m = _depth_param(init_depth_min, B) if torch.is_tensor(init_depth_min) else \
        torch.full((B,), float(init_depth_min), dtype=torch.float32, device=dev)
    if torch.is_tensor(depth_interval):
        step_top = _depth_param(depth_interval, B).to(m.device) * r_top
    else:
        step_top = torch.full((B,), float(depth_interval * r_top), dtype=torch.float32, device=m.device)
    m = m.to(step_top.device)
    far = m + step_top * float(D - 1)
    bad = ~(torch.isfinite(m) & torch.isfinite(far) & (m > 0) & (far > m))
    if m.device.type != "cuda" or not torch.cuda.is_current_stream_capturing():
        if bool(bad.any()):
            i = int(bad.nonzero()[0, 0])
            raise _lib.CasMVSError(
                "inverse depth sampling needs 0 < near < far, both finite: batch item "
                f"{i} has near {float(m[i])}, far {float(far[i])} (init_depth_min, "
                "init_depth_min + (n_depths-1)*depth_interval*ratio of the coarsest stage)")
    u_near = 1.0 / m.double()
    u_far = 1.0 / far.double()
    s_top = (u_near - u_far) / (D - 1)
    steps = [(s_top * interval_ratios[l] / r_top).float() for l in range(top + 1)]
    u_near, u_far = u_near.float(), u_far.float()
    if not tensors:
        return InverseSteps(float(u_near[0]), float(u_far[0]), [float(s[0]) for s in steps], B)
    dev = torch.device(device) if device is not None else m.device
    return InverseSteps(u_near.to(dev), u_far.to(dev), [s.to(dev) for s in steps], B)


def _scalar_or_tensor(x, device):
    """float -> (value, None); tensor -> (0.0, a float32 copy on `device` when it lives elsewhere)."""
    if not torch.is_tensor(x):
        return float(x), None
    return 0.0, x.reshape(-1).to(device=device, dtype=torch.float32).contiguous()


def inverse_hypotheses(steps, level, n_depths, h, w, device, current_depth=None, first_only=False):
    """Planes evenly spaced in inverse depth (README "Wide depth ranges").  current_depth None:
    the coarsest stage, d_k = 1/(u_near - s*k); else current_depth (B,h/2,w/2) is upsampled x2
    and u_0 = max(1/c + (D/2)*s, u_far + (D-1)*s), d_k = 1/(u_0 - s*k).  Returns the depths
    (B,D,h,w), or with first_only=True (finer stages) u_0 (B,h,w), the first rung of an inverse
    Ladder."""
    device = torch.device(device)
    if device.type != "cuda":
        raise _lib.CasMVSError(f"inverse_hypotheses runs on a CUDA device (no CPU fallback); got {device}")
    with torch.cuda.device(device):
        B, D = steps.B, n_depths
        cur = None
        if current_depth is not None:
            _require_cuda(current_depth)
            cur = current_depth.contiguous()
            assert cur.shape == (B, h // 2, w // 2) and cur.device == device
        elif first_only:
            raise _lib.CasMVSError("inverse_hypotheses: first_only needs current_depth (the "
                                   "coarsest stage's first rung is steps.u_near)")
        # steps of CPU tensors (inverse_steps without a device) or of another GPU are copied here
        uf, uf_dev = _scalar_or_tensor(steps.u_near, device)
        ur, ur_dev = _scalar_or_tensor(steps.u_far, device)
        s, s_dev = _scalar_or_tensor(steps.step[level], device)
        planes = 1 if first_only else D
        out = torch.empty((B, h, w) if first_only else (B, D, h, w), device=device, dtype=torch.float32)
        check(_lib.load().casmvs_inverse_hypotheses_fwd(_ptr(cur), uf, _ptr(uf_dev), ur, _ptr(ur_dev), s,
                                                        _ptr(s_dev), _ptr(out), planes, B, D, h, w,
                                                        _stream()), "inverse_hypotheses")
        return out


# --------------------------------------------------------------------------- adaptive depth
# lambda of the adaptive mode: a finer stage searches +-max(lambda*spread, its uniform step)
# around the upsampled depth (UCS-Net's value; kAdaptiveLambda in csrc/regress.cu)
ADAPTIVE_LAMBDA = 1.5


def check_adaptive_depths(n_depths):
    """The adaptive mode spaces D_l planes over a window: every finer stage needs D_l >= 2."""
    for l, D in enumerate(n_depths[:-1]):
        if D < 2:
            raise _lib.CasMVSError(f"adaptive depth sampling needs at least 2 planes in every finer "
                                   f"stage: stage {l} has {D}")


@_on_tensor_device
def adaptive_hypotheses(depth_prev, spread_prev, D, step_l, first_only=False):
    """The planes of a finer stage in the adaptive mode (README "Adaptive depth ranges", rule in
    csrc/regress.cu): depth_prev and spread_prev (B,h/2,w/2) are upsampled x2 to c and s,
    r = max(ADAPTIVE_LAMBDA*s, step_l), lo = max(c - r, 1e-7), hi = c + r, step = (hi - lo)/(D-1)
    and plane k = lo + step*k.  step_l: the stage's uniform step (depth_interval * ratio), a
    float or a (B,)/(B,1) tensor.  Returns the planes (B,D,h,w), or with first_only=True the
    (first, step) maps (B,h,w) of a per-pixel-step Ladder."""
    if D < 2:
        raise _lib.CasMVSError(f"adaptive_hypotheses needs D >= 2 planes (got {D})")
    _require_cuda(depth_prev, spread_prev)
    cur, spr = depth_prev.contiguous(), spread_prev.contiguous()
    B, hi, wi = cur.shape
    assert spr.shape == cur.shape and spr.device == cur.device
    h, w = 2 * hi, 2 * wi
    step, step_dev = _interval_args(step_l, B, cur.device)
    if first_only:
        out = torch.empty(B, h, w, device=cur.device, dtype=torch.float32)
        step_out = torch.empty_like(out)
    else:
        out, step_out = torch.empty(B, D, h, w, device=cur.device, dtype=torch.float32), None
    check(_lib.load().casmvs_adaptive_hypotheses_fwd(_ptr(cur), _ptr(spr), step, _ptr(step_dev), _ptr(out),
                                                     _ptr(step_out), 1 if first_only else D, B, D, h, w,
                                                     _stream()), "adaptive_hypotheses")
    return (out, step_out) if first_only else out


# --------------------------------------------------------------------------- ladder forms
class Ladder:
    """Hypotheses first + step*d of one cascade stage, never materialised as (B,D,h,w):
    `first` is a (B,h,w) tensor [per-pixel], a (B,) tensor [per batch item] or a float; `step` a
    (B,h,w) tensor [per pixel: the adaptive mode; `first` must then be per-pixel too], a (B,)
    tensor or a float; D planes.  `materialize()` gives the tensor the public API takes.
    inverse=True: the ladder is in inverse depth, the hypotheses are 1/(first - step*d) with
    first and step in 1/depth units (inverse_hypotheses)."""

    def __init__(self, first, step, D, B, h, w, device, inverse=False):
        self.first, self.step, self.D, self.B, self.h, self.w, self.device = first, step, D, B, h, w, device
        self.inverse = inverse
        if self.step_map is not None:
            if inverse:
                raise _lib.CasMVSError("Ladder: a per-pixel step is the adaptive mode's, not the inverse mode's")
            if not (torch.is_tensor(first) and first.dim() == 3):
                raise _lib.CasMVSError("Ladder: a per-pixel step needs a per-pixel (B,h,w) first")

    @property
    def step_map(self):
        """The (B,h,w) per-pixel step, or None."""
        return self.step.contiguous() if torch.is_tensor(self.step) and self.step.dim() == 3 else None

    def _args(self):
        fm = fb = sb = None
        f = s = 0.0
        if torch.is_tensor(self.first):
            if self.first.dim() == 3:
                fm = self.first.contiguous()
            else:
                fb = self.first.reshape(-1).contiguous()
        else:
            f = float(self.first)
        if torch.is_tensor(self.step):
            sb = self.step.reshape(-1).contiguous()
        else:
            s = float(self.step)
        return fm, fb, f, sb, s

    def materialize(self):
        d = torch.arange(self.D, device=self.device, dtype=torch.float32).view(1, -1, 1, 1)
        first = self.first if torch.is_tensor(self.first) else torch.tensor(float(self.first), device=self.device)
        step = self.step if torch.is_tensor(self.step) else torch.tensor(float(self.step), device=self.device)
        first = first.view(self.B, 1, self.h, self.w) if first.dim() == 3 else first.reshape(-1, 1, 1, 1)
        if step.dim() == 3:
            return (first + step.view(self.B, 1, self.h, self.w) * d).contiguous()
        if self.inverse:
            u = first - step.reshape(-1, 1, 1, 1) * d
            return torch.reciprocal(u).expand(self.B, self.D, self.h, self.w).contiguous()
        return (first + step.reshape(-1, 1, 1, 1) * d).expand(self.B, self.D, self.h, self.w).contiguous()


def ladder_supported(V, C, num_groups):
    """True when warp_cost_ladder takes this shape: the staged K1 kernel (the only one that takes
    a ladder) covers it.  Otherwise the gather kernel runs from the materialised tensor."""
    return bool(_lib.load().casmvs_warp_cost_ladder_supported(V, C, num_groups))


@_on_tensor_device
def warp_cost_ladder(feats, proj_mats, ladder, num_groups=1, round_tf32=False, blocked=False):
    """warp_cost with the hypotheses given as a Ladder; feats must be channels-last.  Returns the
    logical (B,Cout,D,h,w) channels-last volume, or with blocked=True the (B,Cout/4,D,h,w,4)
    tensor that costreg(blocked=True) takes."""
    _require_cuda(feats, proj_mats)
    _no_grad_only(feats)
    B, V, C, h, w = feats.shape
    assert is_channels_last_feats(feats) and (ladder.B, ladder.h, ladder.w) == (B, h, w)
    cout = C if num_groups == 1 else num_groups
    shape = (B, cout // 4, ladder.D, h, w, 4) if blocked else (B, ladder.D, h, w, cout)
    out = torch.empty(shape, device=feats.device, dtype=torch.float32)
    flags = (1 if round_tf32 else 0) | (BLOCKED if blocked else 0)
    if ladder.step_map is not None:
        check(_lib.load().casmvs_warp_cost_ladder_step_fwd(_ptr(feats), _ptr(proj_mats.contiguous()),
                                                           _ptr(ladder.first.contiguous()), _ptr(ladder.step_map),
                                                           _ptr(out), flags, B, V, C, ladder.D, h, w,
                                                           num_groups, _stream()), "warp_cost_ladder")
        return out if blocked else as_volume_view(out)
    fm, fb, f, sb, s = ladder._args()
    check(_lib.load().casmvs_warp_cost_ladder_fwd(_ptr(feats), _ptr(proj_mats.contiguous()), _ptr(fm),
                                                  _ptr(fb), f, _ptr(sb), s, _ptr(out),
                                                  (1 if round_tf32 else 0) | (BLOCKED if blocked else 0)
                                                  | (INVERSE_DEPTH if ladder.inverse else 0),
                                                  B, V, C, ladder.D, h, w, num_groups, _stream()),
          "warp_cost_ladder")
    return out if blocked else as_volume_view(out)


@_on_tensor_device
def regress_ladder(logits, ladder, want_index=False, want_spread=False):
    """regress over a Ladder -> depth, confidence, index; want_spread=True appends the spread
    (B,h,w) of ops.regress(want_spread=True)."""
    _require_cuda(logits)
    _no_grad_only(logits)
    lg = logits.contiguous()
    B, D, h, w = lg.shape
    depth = torch.empty(B, h, w, device=lg.device, dtype=torch.float32)
    conf = torch.empty_like(depth)
    index = torch.empty(B, h, w, device=lg.device, dtype=torch.int64) if want_index else None
    lib = _lib.load()
    if want_spread or ladder.step_map is not None:
        if want_spread and ladder.inverse:
            raise _lib.CasMVSError("regress_ladder: want_spread is the adaptive mode's, not the inverse mode's")
        spread = torch.empty_like(depth) if want_spread else None
        sm = ladder.step_map
        fm, fb, f, sb, s = (ladder.first.contiguous(), None, 0.0, None, 0.0) if sm is not None else ladder._args()
        check(lib.casmvs_regress_ladder_spread_fwd(_ptr(lg), _ptr(fm), _ptr(fb), f, _ptr(sb), s, _ptr(sm),
                                                   _ptr(depth), _ptr(conf), _ptr(index), _ptr(spread),
                                                   B, D, h, w, _stream()), "regress_ladder")
        return (depth, conf, index, spread) if want_spread else (depth, conf, index)
    fm, fb, f, sb, s = ladder._args()
    fn = lib.casmvs_regress_ladder_inverse_fwd if ladder.inverse else lib.casmvs_regress_ladder_fwd
    check(fn(_ptr(lg), _ptr(fm), _ptr(fb), f, _ptr(sb), s, _ptr(depth), _ptr(conf), _ptr(index),
             B, D, h, w, _stream()), "regress_ladder")
    return depth, conf, index


@_on_tensor_device
def depth_first(current_depth, n_depths, depth_interval):
    """First rung of depth_hypotheses(upsample=True): (B,h/2,w/2) -> (B,h,w)."""
    _require_cuda(current_depth)
    cur = current_depth.contiguous()
    B, hi, wi = cur.shape
    h, w = 2 * hi, 2 * wi
    step, step_dev = _interval_args(depth_interval, B, cur.device)
    half = float(n_depths / 2 * step)
    out = torch.empty(B, h, w, device=cur.device, dtype=torch.float32)
    check(_lib.load().casmvs_depth_first_fwd(_ptr(cur), 1, half, step, _ptr(step_dev), _ptr(out), B,
                                             n_depths, h, w, _stream()), "depth_first")
    return out


# --------------------------------------------------------------------------- FPN (adjacent)
@_on_tensor_device
def fpn_level(prev, c, lat_w, lat_b, smooth_w, smooth_b, want_feat):
    """Fused FeatureNet top-down level (models/mvsnet.py:36-52).  prev (N,32,h/2,w/2),
    c (N,CLAT,h,w) logical NCHW tensors with channels-last storage -> (feat|None, out)."""
    _require_cuda(prev, c, lat_w, lat_b, smooth_w, smooth_b)
    pv = prev.contiguous(memory_format=torch.channels_last)
    cv = c.contiguous(memory_format=torch.channels_last)
    N, clat, h, w = cv.shape
    cout = smooth_w.shape[0]
    assert pv.shape == (N, 32, h // 2, w // 2) and smooth_w.shape[1:] == (32, 3, 3)
    out = torch.empty((N, cout, h, w), device=c.device, dtype=torch.float32,
                      memory_format=torch.channels_last)
    feat = torch.empty((N, 32, h, w), device=c.device, dtype=torch.float32,
                       memory_format=torch.channels_last) if want_feat else None
    check(_lib.load().casmvs_fpn_level_fwd(
        _ptr(pv), _ptr(cv), _ptr(lat_w.detach().contiguous()), _ptr(lat_b.detach().contiguous()),
        _ptr(smooth_w.detach().contiguous()), _ptr(smooth_b.detach().contiguous()), _ptr(feat),
        _ptr(out), N, h, w, clat, cout, _stream()), "fpn_level")
    return feat, out


@_on_tensor_device
def conv2d_planar(x, w_packed, cin, cout, shift=None, slope=1.0, precision=TF32,
                  keep_fp32=False, scale=None):
    """3x3 Conv2d (pad 1) + per-channel scale/shift + LeakyReLU over a channels-last
    (N,Cin,H,W) batch, run as ONE 1x3x3 convolution over the (N,H,W) volume
    (casmvs_conv3d_fwd, kind CONV_PLANAR).  Returns (N,Cout,H,W) channels-last."""
    _require_cuda(x, w_packed, scale, shift)
    _no_grad_only(x)
    xs = x.contiguous(memory_format=torch.channels_last)
    N, C, H, W = xs.shape
    assert C == cin
    y = torch.empty((N, cout, H, W), device=x.device, dtype=torch.float32,
                    memory_format=torch.channels_last)
    check(_lib.load().casmvs_conv3d_fwd(_ptr(xs), _ptr(w_packed), _ptr(scale), _ptr(shift),
                                        float(slope), None, _ptr(y), 1, cin, cout, N, H, W,
                                        CONV_PLANAR, 1,
                                        precision | (KEEP_FP32_OUT if keep_fp32 else 0),
                                        _stream()), "conv2d_planar")
    return y


@_on_tensor_device
def fpn_merge(prev, c, lat_w, lat_b, round_tf32=False):
    """upsample_x2(prev) + conv1x1(c) + bias -> (N,32,h,w) channels-last (prev None: the
    lateral alone, i.e. FeatureNet.toplayer).  models/mvsnet.py:36-47."""
    _require_cuda(prev, c, lat_w, lat_b)
    cv = c.contiguous(memory_format=torch.channels_last)
    N, clat, h, w = cv.shape
    pv = None
    if prev is not None:
        pv = prev.contiguous(memory_format=torch.channels_last)
        assert pv.shape == (N, 32, h // 2, w // 2)
    assert lat_w.shape[0] == 32 and lat_w.shape[1] == clat
    feat = torch.empty((N, 32, h, w), device=c.device, dtype=torch.float32,
                       memory_format=torch.channels_last)
    check(_lib.load().casmvs_fpn_merge_fwd(_ptr(pv), _ptr(cv), _ptr(lat_w.detach().contiguous()),
                                           _ptr(lat_b.detach().contiguous()), _ptr(feat), N, h, w,
                                           clat, 1 if round_tf32 else 0, _stream()), "fpn_merge")
    return feat


@_on_tensor_device
def conv2d_rgb8(x, w, bias, slope, round_tf32=False):
    """First FeatureNet block with folded ABN: planar (N,3,H,W) images -> (N,8,H,W)
    channels-last.  w (8,3,3,3) torch layout."""
    _require_cuda(x, w, bias)
    xs = x.contiguous()
    N, C, H, W = xs.shape
    assert C == 3 and tuple(w.shape) == (8, 3, 3, 3)
    y = torch.empty((N, 8, H, W), device=x.device, dtype=torch.float32,
                    memory_format=torch.channels_last)
    check(_lib.load().casmvs_conv2d_rgb8_fwd(_ptr(xs), _ptr(w.contiguous()), _ptr(bias),
                                             float(slope), _ptr(y), N, H, W,
                                             1 if round_tf32 else 0, _stream()), "conv2d_rgb8")
    return y


@_on_tensor_device
def pack_conv2d_5x5s2_weight(weight):
    """Private copy of a (Cout,Cin,5,5) Conv2d weight for conv2d_5x5s2.  The library caches the
    tensor-core operand image it builds from a weight buffer BY POINTER, so weights must come
    through here (stale images at the new buffer's address are dropped, like pack_conv3d_weight)
    and must not be edited in place."""
    _require_cuda(weight)
    assert weight.dim() == 4 and tuple(weight.shape[2:]) == (5, 5)
    out = torch.empty(weight.shape, device=weight.device, dtype=torch.float32)
    release_weight_images(out)
    out.copy_(weight.detach())
    return out


@_on_tensor_device
def conv2d_5x5s2(x, w, shift, slope, round_tf32=False):
    """5x5 stride-2 pad-2 Conv2d + shift + LeakyReLU on wgmma (FeatureNet conv1.0 / conv2.0
    with folded ABN).  x (N,Cin,H,W) channels-last, w (Cout,Cin,5,5) from
    pack_conv2d_5x5s2_weight -> (N,Cout,H/2,W/2)."""
    _require_cuda(x, w, shift)
    _no_grad_only(x)
    xs = x.contiguous(memory_format=torch.channels_last)
    N, cin, H, W = xs.shape
    cout = w.shape[0]
    assert tuple(w.shape) == (cout, cin, 5, 5) and w.is_contiguous()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = torch.empty((N, cout, Ho, Wo), device=x.device, dtype=torch.float32,
                    memory_format=torch.channels_last)
    check(_lib.load().casmvs_conv2d_5x5s2_fwd(_ptr(xs), _ptr(w), _ptr(shift), float(slope),
                                              _ptr(y), N, cin, cout, H, W,
                                              1 if round_tf32 else 0, _stream()), "conv2d_5x5s2")
    return y


@_on_tensor_device
def conv2d_5x5s2_fp32(x, w, shift, slope):
    """fp32-mode twin of conv2d_5x5s2 (CUDA-core FMA): x (N,Cin,H,W) channels-last,
    w (Cout,Cin,5,5) contiguous -> (N,Cout,H/2,W/2) channels-last."""
    _require_cuda(x, w, shift)
    _no_grad_only(x)
    xs = x.contiguous(memory_format=torch.channels_last)
    N, cin, H, W = xs.shape
    cout = w.shape[0]
    assert tuple(w.shape) == (cout, cin, 5, 5) and w.is_contiguous()
    y = torch.empty((N, cout, (H - 1) // 2 + 1, (W - 1) // 2 + 1), device=x.device,
                    dtype=torch.float32, memory_format=torch.channels_last)
    check(_lib.load().casmvs_conv2d_5x5s2_fp32_fwd(_ptr(xs), _ptr(w), _ptr(shift), float(slope),
                                                   _ptr(y), N, cin, cout, H, W, _stream()),
          "conv2d_5x5s2_fp32")
    return y


@_on_tensor_device
def bias_lrelu_(x, bias, slope, round_tf32=False):
    """In-place LeakyReLU(x + bias[c]) on a channels-last (N,C,h,w) tensor (optionally stored
    TF32-rounded for a tensor-core consumer)."""
    _require_cuda(x, bias)
    assert x.is_contiguous(memory_format=torch.channels_last) and x.shape[1] % 4 == 0
    check(_lib.load().casmvs_bias_act_nhwc(_ptr(x), _ptr(bias), float(slope), x.numel(),
                                           x.shape[1], 1 if round_tf32 else 0, _stream()),
          "bias_lrelu")
    return x


# ------------------------------------------------------------------ DTU point-cloud scoring
def _require_cuda_typed(**tensors):
    """name=(tensor, dtype): CUDA tensors of the given dtypes on one device (no CPU fallback)."""
    first = None
    for name, (t, dtype) in tensors.items():
        if not (torch.is_tensor(t) and t.is_cuda):
            raise _lib.CasMVSError(f"{name} must be a CUDA tensor (no CPU fallback)")
        if t.dtype != dtype:
            raise _lib.CasMVSError(f"{name} must be {dtype}, got {t.dtype}")
        if first is not None and t.device != first.device:
            raise _lib.CasMVSError(f"tensors on different devices: {first.device} and {t.device}")
        if first is None:
            first = t
    _require_cuda(torch.empty(0, device=first.device))


def _points(name, t):
    if not (torch.is_tensor(t) and t.dim() == 2 and t.shape[1] == 3):
        raise _lib.CasMVSError(f"{name} must be an (N,3) tensor")
    if t.shape[0] >= 2 ** 31:
        raise _lib.CasMVSError(f"{name}: at most 2^31 - 1 points")
    return t.contiguous()


@_on_tensor_device
def pcd_cell_keys(points, origin, cell, dims, sub=1):
    """int64 cell key of every point of an (N,3) float32 cloud (casmvs_pcd_cell_keys): cells of
    edge `cell` from `origin`, grid `dims`; sub = 8 orders keys by super cells of 8^3 cells.
    Points outside the grid get the largest int64."""
    pts = _points("points", points)
    _require_cuda_typed(points=(pts, torch.float32))
    keys = torch.empty(pts.shape[0], device=pts.device, dtype=torch.int64)
    ox, oy, oz = (float(v) for v in origin)
    gx, gy, gz = (int(v) for v in dims)
    check(_lib.load().casmvs_pcd_cell_keys(_ptr(pts), pts.shape[0], ox, oy, oz, float(cell),
                                           gx, gy, gz, int(sub), _ptr(keys), _stream()),
          "pcd_cell_keys")
    return keys


@_on_tensor_device
def pcd_thin_prepare(cell_keys, cell_start, n, dims):
    """Workspace of pcd_thin_round for a sub = 1 grid: 27-neighbour table and cell of each point."""
    _require_cuda_typed(cell_keys=(cell_keys, torch.int64), cell_start=(cell_start, torch.int32))
    ncells = cell_keys.shape[0]
    if cell_start.shape[0] != ncells + 1:
        raise _lib.CasMVSError("cell_start must hold ncells + 1 offsets")
    lib = _lib.load()
    nbytes = lib.casmvs_pcd_thin_workspace_bytes(int(n), ncells)
    ws = torch.empty(max(nbytes, 1), device=cell_keys.device, dtype=torch.uint8)
    gx, gy, gz = (int(v) for v in dims)
    check(lib.casmvs_pcd_thin_prepare(_ptr(cell_keys.contiguous()), _ptr(cell_start.contiguous()),
                                      int(n), ncells, gx, gy, gz, _ptr(ws), ws.numel(), _stream()),
          "pcd_thin_prepare")
    return ws


@_on_tensor_device
def pcd_thin_round(points, rank, cell_start, dst, state, undecided, workspace):
    """One join + remove round of the parallel thinning (casmvs_pcd_thin_round); writes the number
    of points still undecided to the device int32 `undecided` (no synchronisation)."""
    pts = _points("points", points)
    _require_cuda_typed(points=(pts, torch.float32), rank=(rank, torch.int32),
                        cell_start=(cell_start, torch.int32), state=(state, torch.uint8),
                        undecided=(undecided, torch.int32), workspace=(workspace, torch.uint8))
    n = pts.shape[0]
    if rank.shape != (n,) or state.shape != (n,) or not state.is_contiguous():
        raise _lib.CasMVSError("rank and state must be contiguous (N,) tensors")
    check(_lib.load().casmvs_pcd_thin_round(
        _ptr(pts), _ptr(rank.contiguous()), _ptr(cell_start.contiguous()), n,
        cell_start.shape[0] - 1, float(dst), _ptr(state), _ptr(undecided), _ptr(workspace),
        workspace.numel(), _stream()), "pcd_thin_round")


@_on_tensor_device
def pcd_capped_nn(queries, targets, cell_keys, cell_start, super_begin, origin, h, super_dims,
                  box_lo, box_hi, cap):
    """min(nearest-target distance, cap) as float64 for queries inside [box_lo, box_hi), cap
    outside (casmvs_pcd_capped_nn).  Targets sorted by their sub = 8 keys; see the header."""
    q = _points("queries", queries)
    t = _points("targets", targets)
    _require_cuda_typed(queries=(q, torch.float32), targets=(t, torch.float32),
                        cell_keys=(cell_keys, torch.int64), cell_start=(cell_start, torch.int32),
                        super_begin=(super_begin, torch.int32))
    ncells = cell_keys.shape[0]
    if cell_start.shape[0] != ncells + 1 or super_begin.shape[0] != math.prod(int(v) for v in super_dims) + 1:
        raise _lib.CasMVSError("cell_start / super_begin sizes do not match the grid")
    dist = torch.empty(q.shape[0], device=q.device, dtype=torch.float64)
    d3 = ctypes.c_double * 3
    check(_lib.load().casmvs_pcd_capped_nn(
        _ptr(q), q.shape[0], _ptr(t), _ptr(cell_keys.contiguous()), _ptr(cell_start.contiguous()),
        ncells, _ptr(super_begin.contiguous()), d3(*map(float, origin)), float(h),
        (ctypes.c_int * 3)(*map(int, super_dims)), d3(*map(float, box_lo)), d3(*map(float, box_hi)),
        float(cap), _ptr(dist), _stream()), "pcd_capped_nn")
    return dist


@_on_tensor_device
def pcd_capped_nn_index(queries, targets, cell_keys, cell_start, super_begin, origin, h, super_dims,
                        box_lo, box_hi, cap, target_index):
    """pcd_capped_nn that also returns the original index (target_index of the key-sorted
    target, int64) of the nearest target, -1 where none lies strictly closer than cap
    (casmvs_pcd_capped_nn_index): -> (dist float64, index int64)."""
    q = _points("queries", queries)
    t = _points("targets", targets)
    _require_cuda_typed(queries=(q, torch.float32), targets=(t, torch.float32),
                        cell_keys=(cell_keys, torch.int64), cell_start=(cell_start, torch.int32),
                        super_begin=(super_begin, torch.int32),
                        target_index=(target_index, torch.int64))
    ncells = cell_keys.shape[0]
    if cell_start.shape[0] != ncells + 1 or super_begin.shape[0] != math.prod(int(v) for v in super_dims) + 1:
        raise _lib.CasMVSError("cell_start / super_begin sizes do not match the grid")
    if target_index.shape != (t.shape[0],):
        raise _lib.CasMVSError("target_index must hold one index per target")
    dist = torch.empty(q.shape[0], device=q.device, dtype=torch.float64)
    index = torch.empty(q.shape[0], device=q.device, dtype=torch.int64)
    d3 = ctypes.c_double * 3
    check(_lib.load().casmvs_pcd_capped_nn_index(
        _ptr(q), q.shape[0], _ptr(t), _ptr(cell_keys.contiguous()), _ptr(cell_start.contiguous()),
        ncells, _ptr(super_begin.contiguous()), d3(*map(float, origin)), float(h),
        (ctypes.c_int * 3)(*map(int, super_dims)), d3(*map(float, box_lo)), d3(*map(float, box_hi)),
        float(cap), _ptr(target_index.contiguous()), _ptr(dist), _ptr(index), _stream()),
          "pcd_capped_nn_index")
    return dist, index


@_on_tensor_device
def pcd_knn_mean(points, k, cell_keys, cell_start, super_begin, origin, h, super_dims, pad,
                 point_index):
    """Mean distance (float64, input order) of every point of a key-sorted (N,3) float32 cloud
    to its k nearest other points (casmvs_pcd_knn_mean); point_index (N,) int64 maps the sorted
    points back to the input order."""
    pts = _points("points", points)
    _require_cuda_typed(points=(pts, torch.float32), cell_keys=(cell_keys, torch.int64),
                        cell_start=(cell_start, torch.int32), super_begin=(super_begin, torch.int32),
                        point_index=(point_index, torch.int64))
    ncells = cell_keys.shape[0]
    if cell_start.shape[0] != ncells + 1 or super_begin.shape[0] != math.prod(int(v) for v in super_dims) + 1:
        raise _lib.CasMVSError("cell_start / super_begin sizes do not match the grid")
    if point_index.shape != (pts.shape[0],):
        raise _lib.CasMVSError("point_index must hold one index per point")
    mean = torch.empty(pts.shape[0], device=pts.device, dtype=torch.float64)
    check(_lib.load().casmvs_pcd_knn_mean(
        _ptr(pts), pts.shape[0], int(k), _ptr(cell_keys.contiguous()), _ptr(cell_start.contiguous()),
        ncells, _ptr(super_begin.contiguous()), (ctypes.c_double * 3)(*map(float, origin)), float(h),
        (ctypes.c_int * 3)(*map(int, super_dims)), float(pad), _ptr(point_index.contiguous()),
        _ptr(mean), _stream()), "pcd_knn_mean")
    return mean


@_on_tensor_device
def pcd_sor_keep(mean, std_ratio):
    """Statistics and keep mask of (N,) float64 mean distances (casmvs_pcd_sor_keep) ->
    (stats (3,) float64 device tensor mu, sigma, threshold; mask (N,) uint8; block counts (int32,
    as tnt_compact takes them); chunk sums (2, ceil(N / 1024)) float64)."""
    _require_cuda_typed(mean=(mean, torch.float64))
    m = mean.contiguous()
    n = m.shape[0]
    lib = _lib.load()
    nbytes = lib.casmvs_pcd_sor_workspace_bytes(n)
    ws = torch.empty(max(nbytes // 8, 2), device=m.device, dtype=torch.float64)
    stats = torch.empty(3, device=m.device, dtype=torch.float64)
    mask = torch.empty(n, device=m.device, dtype=torch.uint8)
    counts = torch.empty(max(lib.casmvs_tnt_crop_blocks(n), 1), device=m.device, dtype=torch.int32)
    check(lib.casmvs_pcd_sor_keep(_ptr(m), n, float(std_ratio), _ptr(stats), _ptr(mask),
                                  _ptr(counts), _ptr(ws), nbytes, _stream()), "pcd_sor_keep")
    return stats, mask, counts, ws.view(2, -1)


# ------------------------------------------------------------------ Tanks and Temples scoring
@_on_tensor_device
def tnt_transform_crop(points, T=None, crop=None):
    """float32(T p) of every point of an (N,3) float32 cloud (casmvs_tnt_transform_crop; T a 4x4
    or None for the points as they are).  With crop = (axis, axis_min, axis_max, polygon (m,2)
    float64 CUDA tensor of (u, v) vertices) -> the transformed points inside the crop volume in
    input order and their input indices (int64); without -> the transformed points."""
    pts = _points("points", points)
    _require_cuda_typed(points=(pts, torch.float32))
    n = pts.shape[0]
    lib = _lib.load()
    out = torch.empty_like(pts)
    Tp = None
    if T is not None:
        rows = torch.as_tensor(T, dtype=torch.float64).reshape(4, 4)[:3].reshape(-1).tolist()
        Tp = (ctypes.c_double * 12)(*rows)
    if crop is None:
        check(lib.casmvs_tnt_transform_crop(_ptr(pts), n, Tp, -1, 0.0, 0.0, None, 0, _ptr(out),
                                            None, None, _stream()), "tnt_transform_crop")
        return out
    axis, amin, amax, poly = crop
    _require_cuda_typed(points=(pts, torch.float32), polygon=(poly, torch.float64))
    poly = poly.contiguous()
    if poly.dim() != 2 or poly.shape[1] != 2:
        raise _lib.CasMVSError("polygon must be an (m,2) tensor")
    nb = lib.casmvs_tnt_crop_blocks(n)
    mask = torch.empty(n, device=pts.device, dtype=torch.uint8)
    counts = torch.empty(max(nb, 1), device=pts.device, dtype=torch.int32)
    check(lib.casmvs_tnt_transform_crop(_ptr(pts), n, Tp, int(axis), float(amin), float(amax),
                                        _ptr(poly), poly.shape[0], _ptr(out), _ptr(mask),
                                        _ptr(counts), _stream()), "tnt_transform_crop")
    return tnt_compact(out, mask, counts)


@_on_tensor_device
def tnt_compact(points, mask, block_counts):
    """The points with mask != 0 in input order and their input indices (int64), given the kept
    count of each block of casmvs_tnt_crop_blocks(N) (casmvs_tnt_compact)."""
    pts = _points("points", points)
    _require_cuda_typed(points=(pts, torch.float32), mask=(mask, torch.uint8),
                        block_counts=(block_counts, torch.int32))
    n = pts.shape[0]
    lib = _lib.load()
    nb = lib.casmvs_tnt_crop_blocks(n)
    if mask.shape != (n,) or block_counts.numel() < nb:
        raise _lib.CasMVSError("mask must hold one entry per point and block_counts one per block")
    offsets = torch.zeros(max(nb, 1) + 1, device=pts.device, dtype=torch.int64)
    torch.cumsum(block_counts[:nb], 0, out=offsets[1:nb + 1])
    kept = int(offsets[nb].item()) if nb else 0
    res = torch.empty((kept, 3), device=pts.device, dtype=torch.float32)
    idx = torch.empty(kept, device=pts.device, dtype=torch.int64)
    check(lib.casmvs_tnt_compact(_ptr(pts), _ptr(mask.contiguous()), n, _ptr(offsets), _ptr(res),
                                 _ptr(idx), _stream()), "tnt_compact")
    return res, idx


@_on_tensor_device
def tnt_voxel_mean(points, order, voxel_start):
    """float32 mean of each voxel's points order[voxel_start[v]:voxel_start[v+1]], summed in double
    in that order (casmvs_tnt_voxel_mean)."""
    pts = _points("points", points)
    _require_cuda_typed(points=(pts, torch.float32), order=(order, torch.int64),
                        voxel_start=(voxel_start, torch.int32))
    nv = voxel_start.shape[0] - 1
    out = torch.empty((max(nv, 0), 3), device=pts.device, dtype=torch.float32)
    check(_lib.load().casmvs_tnt_voxel_mean(_ptr(pts), _ptr(order.contiguous()),
                                            _ptr(voxel_start.contiguous()), max(nv, 0), _ptr(out),
                                            _stream()), "tnt_voxel_mean")
    return out


@_on_tensor_device
def tnt_icp_moments(src, tgt, index, origin):
    """The 18 float64 correspondence moments of casmvs_tnt_icp_moments (device tensor):
    count, sum d^2, sum s', sum t', sum |s'|^2, sum t' s'^T (row-major) about `origin`."""
    s = _points("src", src)
    t = _points("tgt", tgt)
    _require_cuda_typed(src=(s, torch.float32), tgt=(t, torch.float32), index=(index, torch.int64))
    if index.shape != (s.shape[0],):
        raise _lib.CasMVSError("index must hold one entry per source point")
    lib = _lib.load()
    n = s.shape[0]
    nbytes = lib.casmvs_tnt_icp_workspace_bytes(n)
    ws = torch.empty(nbytes // 8, device=s.device, dtype=torch.float64)
    out = torch.empty(18, device=s.device, dtype=torch.float64)
    check(lib.casmvs_tnt_icp_moments(_ptr(s), n, _ptr(t), _ptr(index.contiguous()),
                                     (ctypes.c_double * 3)(*map(float, origin)), _ptr(out), _ptr(ws),
                                     nbytes, _stream()), "tnt_icp_moments")
    return out
