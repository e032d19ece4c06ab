"""Adaptive depth ranges (csrc/regress.cu, README "Adaptive depth ranges") restated:

  * hypotheses_f32: rule 3 with one float32 rounding per operation, in the kernel's order
    (numpy).  adaptive_hypotheses and a per-pixel-step Ladder's materialize() must equal it bit
    for bit; hypotheses_f64 is the same rule in float64 from the same upsampled inputs;
  * spread_ref: rule 2 in float64, sigma = sqrt(sum_k p_k (d_k - dhat)^2), with a per-element
    bound built on regress_fp64's bounds of p and dhat;
  * cascade_forward_adaptive: the cascade oracle (casmvs_oracle) with the adaptive planes at the
    finer stages.  The uniform cascade_forward stays the default.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import casmvs_oracle as O
from . import regress_fp64 as RG
from .inverse_depth_fp64 import upsample_f32

f32 = np.float32
LAMBDA = 1.5                     # ops.ADAPTIVE_LAMBDA / kAdaptiveLambda
THRESH = f32(1e-7)
ULP = 2.0 ** -24


def _steps(step_l, B):
    if torch.is_tensor(step_l):
        a = step_l.detach().reshape(-1).cpu().numpy().astype(f32)
        return np.broadcast_to(a, (B,)) if a.size == 1 else a
    return np.full(B, f32(step_l), dtype=f32)


def _np32(x):
    return x.detach().cpu().numpy().astype(f32) if torch.is_tensor(x) else np.asarray(x, dtype=f32)


def window_f32(cur, spread, D, step_l):
    """Rule 3 up to the ladder: -> lo, step (B,h,w) float32.  cur, spread (B,h/2,w/2)."""
    cur, spread = _np32(cur), _np32(spread)
    B = cur.shape[0]
    g = _steps(step_l, B).reshape(-1, 1, 1)
    c = upsample_f32(cur)
    s = upsample_f32(spread)
    with np.errstate(invalid="ignore", over="ignore"):
        ls = (f32(LAMBDA) * s).astype(f32)
        r = np.fmax(ls, g).astype(f32)               # fmax ignores NaN, as fmaxf does
        lo = np.fmax((c - r).astype(f32), THRESH).astype(f32)
        hi = (c + r).astype(f32)
        step = ((hi - lo).astype(f32) / f32(D - 1)).astype(f32)
    return lo, step


def hypotheses_f32(cur, spread, D, step_l, first_only=False):
    """-> the planes (B,D,h,w) RN(lo + RN(step*k)), or with first_only the (lo, step) maps."""
    lo, step = window_f32(cur, spread, D, step_l)
    if first_only:
        return lo, step
    k = np.arange(D, dtype=f32).reshape(1, -1, 1, 1)
    with np.errstate(invalid="ignore", over="ignore"):
        return (lo[:, None] + (step[:, None] * k).astype(f32)).astype(f32)


def hypotheses_f64(cur, spread, D, step_l):
    """Rule 3 in float64 from the same float32 upsampled c and s -> (B,D,h,w) float64."""
    cur, spread = _np32(cur), _np32(spread)
    B = cur.shape[0]
    g = _steps(step_l, B).reshape(-1, 1, 1).astype(np.float64)
    c = upsample_f32(cur).astype(np.float64)
    s = upsample_f32(spread).astype(np.float64)
    r = np.fmax(LAMBDA * s, g)
    lo = np.fmax(c - r, float(THRESH))
    hi = c + r
    k = np.arange(D, dtype=np.float64).reshape(1, -1, 1, 1)
    return lo[:, None] + (hi - lo)[:, None] / (D - 1) * k


def ladder_f32(first, step, D):
    """The planes of a per-pixel-step Ladder: first, step (B,h,w) -> RN(first + RN(step*k))."""
    fa, sa = _np32(first), _np32(step)
    k = np.arange(D, dtype=f32).reshape(1, -1, 1, 1)
    return (fa[:, None] + (sa[:, None] * k).astype(f32)).astype(f32)


@torch.no_grad()
def spread_ref(logits, hyp, input_is_prob=False, eps=2.0 ** -17):
    """Rule 2 in float64 -> sigma64 (B,h,w), bound (B,h,w).

    With p and dhat the float64 regression and dp, Dl their bounds (regress_fp64.regress_ref, eps
    included), e_k = d_k - dhat: the kernel's t_k = RN(d_k - dhat~) satisfies |t_k| <= E_k =
    (|e_k| + Dl)(1 + u), RN(t_k^2) adds u, the product u and the Cascade16 sum eps relative, so
        |var~ - var64| <= b = (sum dp E^2 + sum p (E^2 - e^2 + 3u E^2) + eps sum (p + dp) E^2) SAFE,
    and sigma = sqrt_rn(var~) is within min(sqrt(b), b / (sigma64 + sqrt(max(var64 - b, 0))))
    of sigma64, plus half an ulp of the result."""
    ref = RG.regress_ref(logits, hyp, input_is_prob)
    p = ref["p"]
    dp = ref["dp0"] + eps * ref["pA"]
    dhat = ref["depth"].unsqueeze(1)
    Dl = (ref["depth_b0"] + eps * ref["depth_A"]).unsqueeze(1)
    dv = RG._dv(hyp, p)
    e = dv - dhat
    E = (e.abs() + Dl) * (1 + ULP)
    var64 = (p * e * e).sum(1)
    b = ((dp * E * E).sum(1) + (p * (E * E - e * e + 3 * ULP * E * E)).sum(1)
         + eps * ((p + dp) * E * E).sum(1)) * RG.SAFE
    sig = var64.sqrt()
    den = sig + (var64 - b).clamp_min(0).sqrt()
    lin = torch.where(den > 0, b / den, torch.full_like(b, float("inf")))
    bound = torch.minimum(b.sqrt(), lin)
    return sig, bound + ULP * (sig + bound)


def cascade_forward_adaptive(sd, imgs, proj_mats, init_depth_min, depth_interval,
                             n_depths=(8, 32, 48), interval_ratios=(1, 2, 4), num_groups=1):
    """casmvs_oracle.cascade_forward with the adaptive planes (rules 1-3), on CPU in the dtype of
    its inputs as cascade_forward runs.  Returns depth, confidence, index and, for the stages
    that write one, the spread."""
    B, V = imgs.shape[:2]
    H, W = imgs.shape[-2:]
    dt = imgs.dtype
    top = len(n_depths) - 1
    results = {}
    with torch.no_grad():
        feats = O.feature_pyramid(imgs.reshape(B * V, 3, H, W), sd)
        depth_l = spread_l = None
        for l in range(top, -1, -1):
            f = feats[f"level_{l}"]
            f = f.reshape(B, V, *f.shape[1:])
            D = n_depths[l]
            h, w = f.shape[-2:]
            interval_l = depth_interval * interval_ratios[l]
            if l == top:
                dv = O.initial_hypotheses(init_depth_min, interval_l, D, B, h, w).to(dt)
            else:
                g = interval_l.to(dt).reshape(-1, 1, 1, 1) if torch.is_tensor(interval_l) else interval_l
                c = O.upsample_depth(depth_l)
                s = O.upsample_depth(spread_l)
                r = torch.fmax(LAMBDA * s, torch.as_tensor(g, dtype=dt).expand_as(s))
                lo = torch.fmax(c - r, torch.tensor(float(THRESH), dtype=dt))
                hi = c + r
                k = torch.arange(D, dtype=dt).reshape(1, -1, 1, 1)
                dv = lo + (hi - lo) / (D - 1) * k
            if num_groups == 1:
                cost = O.variance_cost_volume(f, proj_mats[:, :, l], dv)
            else:
                cost = O.groupwise_cost_volume(f, proj_mats[:, :, l], dv, num_groups)
            logits = O.cost_regularize(cost, sd, f"cost_reg_{l}.").squeeze(1)
            depth_l, conf_l, index_l, p = O.regress_depth(logits, dv)
            spread_l = (p * (dv - depth_l.unsqueeze(1)) ** 2).sum(1).sqrt()
            results[f"depth_{l}"] = depth_l
            results[f"confidence_{l}"] = conf_l
            results[f"depth_index_{l}"] = index_l
            if l > 0:
                results[f"spread_{l}"] = spread_l
            results[f"hypotheses_{l}"] = dv
    return results
