"""Float64 reference of depth regression (K3, csrc/regress.cu), its backward
(casmvs_regress_bwd) and the depth hypotheses (K4), with a per-element error bound, for
per-element checks.

Plain torch only (no casmvsnet_pl_b200 import): the module takes the float32 logits and
hypotheses the kernel sees.  A ladder first + step*d is passed materialised
(``ops.Ladder.materialize()`` rounds like the kernels: the product, then the sum).  Tensors:
logits and hypotheses (B, D, h, w), or hypotheses (D,); maps (B, h, w).

Bounds, derived from the kernels' fp32 arithmetic (u = 2^-24, SAFE = 1 + 2^-20 for second-order
terms); eps is the measured relative error of the kernels' fp32 reductions:

* Probabilities.  p64 = softmax(l) in float64.  The kernel's exp(l_d - m) has relative error
  delta_d = expm1(a_d) + 4u exp(a_d), a_d = |fl(l_d - m) - (l_d - m)| the error of the rounded
  argument (one IEEE subtraction of float32 values, so the oracle evaluates it exactly; at most
  u |l_d - m|) and 4u for expf (2 ulp; the library is built without fast-math), plus ABS_E
  absolute where it underflows.  Its sequential denominator of positive terms carries
  sum_j p64_j delta_j (the inputs) and eps (the reduction) relative, the IEEE division u, so
      |p - p64| <= p64 (delta_d + sum_j p64_j delta_j + u) SAFE + (D + 2) ABS_E  +  eps p64.
  input_is_prob: p is the input, exact.
* Depth and fidx.  depth = sum_d p_d dv_d and fidx = sum_d p_d d (rounded products, Cascade16
  sums): |depth - depth64| <= sum |dp| |dv| + u sum p |dv| + eps sum p |dv|, where dp's eps term
  is counted in A too: A = sum p |dv| (the sum) + sum p |dv| (the denominator inside each p).
* Index.  The kernel truncates fidx and clamps it to [0, D-1].  Where fidx64 lies farther than
  its bound from every integer k in [1, D-1] the index must be clamp(trunc(fidx64), 0, D-1);
  within that distance of k, k - 1 and k are both accepted (``ambiguous``).
* Confidence.  The sum of p over the window [idx-1, idx+2] at the kernel's own index, zero
  padded: bound sum |dp| over the window, A = 2 sum p (4-term sum and denominator).
* Backward.  d depth / d l_d = p_d (dv_d - depth): the kernel recomputes depth = num / den
  (an fma chain and a sequential sum), then e_d (dv_d - depth) (g / den).  With
  ddepth = sum p delta |dv| + (sum p delta + u) |depth64|,
      bound0 = |g| p64 (ddepth + |dv - depth64| (delta_d + sum p delta + 4u)) SAFE,
      A = |g| p64 (sum p |dv| + |depth64| + |dv - depth64|).
* Inverse mode (README "Wide depth ranges", regress.cu rule 5).  The kernels average
  v_d = RN(1/dv_d), one IEEE float32 division the oracle takes exactly, so ubar = sum p_d v_d
  carries the depth bound above with dv replaced by v.  depth = RN(1/ubar): with Dl = that bound
  (eps included), |1/ubar~ - 1/ubar| <= Dl / (ubar (ubar - Dl)) = depth64^2 Dl ubar / (ubar - Dl),
  plus half an ulp of the depth.  Index and confidence are the uniform mode's.
  Backward: d depth / d l_d = -depth^2 p_d (v_d - ubar): the uniform bound of p_d (v_d - ubar) g
  (regress_inv_bwd_kernel forms ubar = num / den as the uniform kernel forms its depth), scaled
  by depth64^2, plus that term times the relative error of the kernel's depth^2: twice ubar's
  (ddepth / ubar above, and 2 eps for its two sums) plus 4u (the reciprocal, the square and the
  two products with it).
* K4.  first = max(up(cur) - half, 1e-7f), out = first + step d.  up is the upsample of
  oracle/feature_fp64.py (position and blend bound); half = D/2 step is rounded once (the
  scalar path also rounds step itself: 2u |half|); the subtraction, the product and the sum add
  u each.  No reduction, so no eps.  Where even the bound keeps up(cur) - half below 1e-7 the
  first rung is exactly 1e-7f.
"""
from __future__ import annotations

import torch

from oracle import feature_fp64 as FF
from oracle.conv3d_fp64 import TINY  # noqa: F401

ULP = 2.0 ** -24
SAFE = FF.SAFE
EXP_REL = 4 * ULP                    # expf: 2 ulp
ABS_E = 2.0 ** -147                  # expf near underflow: 2 ulp of the subnormal spacing
THRESH = float(torch.tensor(1e-7, dtype=torch.float32))


def _dv(hyp, like):
    dv = hyp.to(device=like.device, dtype=torch.float64)
    return dv.view(1, -1, 1, 1) if dv.dim() == 1 else dv


def inverse_values(hyp):
    """v = RN(1/hyp) in float32: what the inverse-mode kernels average (plane_value<true>)."""
    return torch.div(1.0, hyp.detach().cpu().float()).to(hyp.device)


def softmax_ref(logits, input_is_prob=False):
    """-> p64, its bound without eps dp0, the per-plane relative error delta of exp, and
    theta = sum p64 delta (all (B, D, h, w) but theta (B, 1, h, w))."""
    l = logits.double()
    if input_is_prob:
        z = torch.zeros_like(l)
        return l, z, z, z[:, :1]
    m = logits.amax(1, keepdim=True)
    t = l - m.double()
    e = t.exp()
    p = e / e.sum(1, keepdim=True)
    # the kernels' argument fl(l - m) is one IEEE subtraction: its error is known exactly
    da = ((logits - m).double() - t).abs()
    delta = (torch.expm1(da) + EXP_REL * torch.exp(da)) * SAFE
    theta = (p * delta).sum(1, keepdim=True)
    D = l.shape[1]
    dp0 = p * (delta + theta + ULP) * SAFE + ABS_E * (D + 2)
    return p, dp0, delta, theta


def regress_ref(logits, hyp, input_is_prob=False, inverse=False):
    """Float64 K3 without the index decision: dict of p, dp0, pA (the eps magnitude of p),
    depth / fidx with their bound0 and A.  inverse: 'depth' is ubar = sum p RN(1/hyp), the
    average before the final reciprocal."""
    if inverse:
        hyp = inverse_values(hyp)
    p, dp0, _, _ = softmax_ref(logits, input_is_prob)
    pA = torch.zeros_like(p) if input_is_prob else p
    dv = _dv(hyp, p)
    D = p.shape[1]
    dd = torch.arange(D, dtype=torch.float64, device=p.device).view(1, D, 1, 1)
    out = dict(p=p, dp0=dp0, pA=pA)
    for name, v in (("depth", dv), ("fidx", dd)):
        s = (p * v.abs()).sum(1)
        out[name] = (p * v).sum(1)
        out[name + "_b0"] = (dp0 * v.abs()).sum(1) + ULP * s * SAFE
        out[name + "_A"] = s + (pA * v.abs()).sum(1)
    return out


def index_check(index, fidx64, fidx_bound, D):
    """-> (ok map, ambiguous map): the kernel's index against clamp(trunc(fidx64), 0, D-1),
    either neighbour of an integer k in [1, D-1] accepted within the bound of k."""
    idx = index.to(device=fidx64.device)
    want = fidx64.trunc().clamp(0, D - 1).long()
    k = fidx64.round()
    amb = (k >= 1) & (k <= D - 1) & ((fidx64 - k).abs() <= fidx_bound)
    kl = k.long()
    ok = (idx == want) | (amb & ((idx == kl) | (idx == kl - 1)))
    return ok, amb


def confidence_ref(ref, index):
    """Float64 sum of p over [idx-1, idx+2] at the kernel's index (zero padded) -> c64, bound0,
    A."""
    p, dp0, pA = ref["p"], ref["dp0"], ref["pA"]
    B, D, h, w = p.shape
    idx = index.to(device=p.device).long().unsqueeze(1)
    c = torch.zeros(B, 1, h, w, dtype=torch.float64, device=p.device)
    b0, A = torch.zeros_like(c), torch.zeros_like(c)
    for k in (-1, 0, 1, 2):
        d = idx + k
        inside = (d >= 0) & (d < D)
        dc = d.clamp(0, D - 1)
        for acc, t in ((c, p), (b0, dp0), (A, p + pA)):
            acc += torch.where(inside, t.gather(1, dc), torch.zeros_like(c))
    return c[:, 0], b0[:, 0], A[:, 0]


def regress_bwd_ref(logits, hyp, gdepth, inverse=False):
    """Float64 gradient of sum(depth * gdepth) with respect to the logits: (B, D, h, w) g64,
    bound0, A.  inverse: the inverse regression's, -depth^2 p (RN(1/hyp) - ubar) gdepth."""
    if inverse:
        hyp = inverse_values(hyp)
    p, _, delta, theta = softmax_ref(logits)
    dv = _dv(hyp, p)
    depth = (p * dv).sum(1, keepdim=True)
    sabs = (p * dv.abs()).sum(1, keepdim=True)
    diff = dv - depth
    g = gdepth.to(device=p.device, dtype=torch.float64).unsqueeze(1)
    ddepth = (p * delta * dv.abs()).sum(1, keepdim=True) + (theta + ULP) * depth.abs()
    b0 = g.abs() * p * (ddepth + diff.abs() * (delta + theta + 4 * ULP)) * SAFE
    b0 = b0 + g.abs() * ABS_E * (p.shape[1] + 2) * (dv.abs() + depth.abs())
    A = g.abs() * p * (sabs + depth.abs() + diff.abs())
    gu = g * p * diff
    if not inverse:
        return gu, b0, A
    dep2 = depth ** -2                                     # depth = ubar here
    rel = 2 * ddepth / depth.abs() + 4 * ULP
    # SAFE once more: the product of depth^2's relative error with the error b0 already bounds
    # is second order
    return -dep2 * gu, dep2 * (b0 + gu.abs() * rel) * SAFE, dep2 * (A + 4 * gu.abs())


# ------------------------------------------------------------------------------- K4
def _per_item(v, B, device):
    t = torch.as_tensor(v, dtype=torch.float64, device=device).reshape(-1)
    return (t.expand(B) if t.numel() == 1 else t).view(B, 1, 1, 1)


def hypotheses_ref(cur, D, step, upsample):
    """depth_hypotheses / depth_first: cur (B, h/2, w/2) with upsample, else (B, 1, h, w) or
    (B, h, w); step the float32 value(s) the kernel uses (float, or (B,) / (B, 1)).
    -> out64 (B, D, h, w), bound, clamped (B, h, w): where the first rung is exactly 1e-7f."""
    B = cur.shape[0]
    if upsample:
        c, cb0, _ = FF.upsample2x(cur.unsqueeze(-1))
        c, cb0 = c[..., 0], cb0[..., 0]
    else:
        c = cur.double().reshape(B, *cur.shape[-2:])
        cb0 = torch.zeros_like(c)
    c, cb0 = c.unsqueeze(1), cb0.unsqueeze(1)
    s = _per_item(step, B, c.device)
    half = D / 2 * s
    a = c - half
    da = cb0 + (2 * ULP * half.abs() + ULP * a.abs()) * SAFE
    first = a.clamp_min(THRESH)
    d = torch.arange(D, dtype=torch.float64, device=c.device).view(1, D, 1, 1)
    sd = s * d
    out = first + sd
    bound = (da + ULP * sd.abs() + ULP * out.abs()) * SAFE + TINY
    clamped = (a + da < THRESH)[:, 0]
    return out, bound, clamped


def uniform_ref(depth_min, step, B, D, h, w, device="cpu"):
    """uniform_hypotheses from the float32 value(s) of depth_min and step -> out64, bound."""
    dm, s = _per_item(depth_min, B, device), _per_item(step, B, device)
    d = torch.arange(D, dtype=torch.float64, device=device).view(1, D, 1, 1)
    out = (dm + s * d).expand(B, D, h, w)
    bound = (ULP * (s * d).abs() + ULP * out.abs()) * SAFE + TINY
    return out, bound


# ------------------------------------------------------------------------------- reports
Report = FF.Report


@torch.no_grad()
def check(y, y64, bound0, A, eps, names, scale=None):
    rep = Report(eps, False, names)
    rep.add(y, y64, bound0, A, (0,) * y64.dim(), A if scale is None else scale)
    return rep


@torch.no_grad()
def check_regress(logits, hyp, depth, conf, index=None, prob=None, input_is_prob=False,
                  eps=2.0 ** -17, inverse=False):
    """Every output of one K3 call against float64 -> dict of Reports ('prob', 'depth',
    'conf') plus 'index': (number of wrong pixels, number of ambiguous pixels, first wrong
    (b, y, x) or None).  inverse: the call regressed in 1/depth (regress(..., inverse=True))."""
    ref = regress_ref(logits, hyp, input_is_prob, inverse)
    if inverse:
        u, ub0, uA = ref["depth"], ref["depth_b0"], ref["depth_A"]
        dl = ub0 + eps * uA
        # a bound as large as ubar itself cannot be carried through 1/ubar: infinite there
        grow = torch.where(dl < u, u / (u - dl), torch.full_like(u, float("inf")))
        d64 = 1.0 / u
        ref["depth"] = d64
        ref["depth_b0"] = d64 ** 2 * ub0 * grow + ULP * d64
        ref["depth_A"] = d64 ** 2 * uA * grow
    D = logits.shape[1]
    out = {}
    names3 = ("b", "y", "x")
    if prob is not None:
        out["prob"] = check(prob, ref["p"], ref["dp0"], ref["pA"], eps, ("b", "d", "y", "x"),
                            scale=ref["p"])
    out["depth"] = check(depth, ref["depth"], ref["depth_b0"], ref["depth_A"], eps, names3)
    fb = ref["fidx_b0"] + eps * ref["fidx_A"]
    if index is not None:
        ok, amb = index_check(index, ref["fidx"], fb, D)
        bad = (~ok).nonzero()
        out["index"] = (int(bad.shape[0]), int(amb.sum()),
                        tuple(int(v) for v in bad[0]) if bad.shape[0] else None)
        idx = index
    else:
        idx = ref["fidx"].trunc().clamp(0, D - 1).long()
    c64, cb0, cA = confidence_ref(ref, idx)
    out["conf"] = check(conf, c64, cb0, cA, eps, names3)
    return out
