"""The inverse-depth plane sweep (csrc/regress.cu, README "Wide depth ranges") restated:

  * steps_f32: rules 1-2, the far plane in float32 and the inverse steps in float64, each
    rounded once to float32;
  * hypotheses_f32 / first_rung_f32: rules 3-4 with one float32 rounding per operation, in the
    kernels' order (numpy).  The kernels must equal these bit for bit;
  * ladder_f32: the depths of an inverse ladder (first, step), the same way: the hypotheses the
    K1 and K3 checks give their float64 references for a ladder call;
  * regress_f64 / regress_bwd_f64: rule 5 and its backward in float64;
  * cascade_forward_inverse: the cascade oracle (casmvs_oracle) with inverse hypotheses and the
    inverse regression.  The uniform cascade_forward stays the default.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import casmvs_oracle as O

f32 = np.float32


def _per_item(x, B):
    if torch.is_tensor(x):
        a = x.detach().reshape(-1).cpu().numpy()
        return np.broadcast_to(a, (B,)) if a.size == 1 else a
    return np.full(B, x, dtype=np.float64)


def steps_f32(init_depth_min, depth_interval, n_depths, ratios, B):
    """Rules 1-2 -> (u_near, u_far, [s_l]), float32 arrays (B,); raises ValueError on rule 1."""
    top = len(n_depths) - 1
    D, r_top = n_depths[top], ratios[top]
    m = _per_item(init_depth_min, B).astype(f32)
    if torch.is_tensor(depth_interval):
        st = (_per_item(depth_interval, B).astype(f32) * f32(r_top)).astype(f32)
    else:
        st = np.full(B, f32(depth_interval * r_top), dtype=f32)
    far = (m + (st * f32(D - 1)).astype(f32)).astype(f32)
    ok = np.isfinite(m) & np.isfinite(far) & (m > 0) & (far > m)
    if not ok.all():
        raise ValueError("inverse depth sampling needs 0 < near < far, both finite")
    un = 1.0 / m.astype(np.float64)
    uf = 1.0 / far.astype(np.float64)
    s_top = (un - uf) / (D - 1)
    return un.astype(f32), uf.astype(f32), [(s_top * ratios[l] / r_top).astype(f32)
                                            for l in range(top + 1)]


def _rcp(x):
    return (f32(1.0) / x.astype(f32)).astype(f32)


def upsample_f32(cur):
    """The kernels' x2 bilinear (align_corners=True) of a (B,hi,wi) float32 array, operation by
    operation as upsample2x_at forms it."""
    B, hi, wi = cur.shape
    h, w = 2 * hi, 2 * wi
    sy = f32(hi - 1) / f32(h - 1) if hi > 1 else f32(0)
    sx = f32(wi - 1) / f32(w - 1) if wi > 1 else f32(0)
    fy = (f32(sy) * np.arange(h, dtype=f32)).astype(f32)
    fx = (f32(sx) * np.arange(w, dtype=f32)).astype(f32)
    y0 = np.minimum(fy.astype(np.int64), hi - 1)
    x0 = np.minimum(fx.astype(np.int64), wi - 1)
    y1, x1 = np.minimum(y0 + 1, hi - 1), np.minimum(x0 + 1, wi - 1)
    ly = (fy - y0.astype(f32)).astype(f32)[:, None]
    lx = (fx - x0.astype(f32)).astype(f32)[None, :]
    c = cur.astype(f32)
    v00, v01 = c[:, y0][:, :, x0], c[:, y0][:, :, x1]
    v10, v11 = c[:, y1][:, :, x0], c[:, y1][:, :, x1]
    ilx, ily = (f32(1) - lx).astype(f32), (f32(1) - ly).astype(f32)
    top = ((ilx * v00).astype(f32) + (lx * v01).astype(f32)).astype(f32)
    bot = ((ilx * v10).astype(f32) + (lx * v11).astype(f32)).astype(f32)
    return ((ily * top).astype(f32) + (ly * bot).astype(f32)).astype(f32)


def first_rung_f32(steps, level, D, cur):
    """u_0 (B,h,w): u_near for the coarsest stage (cur None), else rule 4's clamp."""
    un, uf, s = steps[0], steps[1], steps[2][level]
    if cur is None:
        return un.reshape(-1, 1, 1)
    uc = _rcp(upsample_f32(cur))
    sb = s.reshape(-1, 1, 1)
    a = (uc + (f32(D * 0.5) * sb).astype(f32)).astype(f32)
    b = (uf.reshape(-1, 1, 1) + (f32(D - 1) * sb).astype(f32)).astype(f32)
    return np.maximum(a, b).astype(f32)


def hypotheses_f32(steps, level, D, h, w, cur=None):
    """Rules 3-4 -> (B,D,h,w) float32 depths d_k = RN(1/(u_0 - s*k))."""
    u0 = np.broadcast_to(first_rung_f32(steps, level, D, cur), (len(steps[0]), h, w))
    s = steps[2][level].reshape(-1, 1, 1, 1)
    k = np.arange(D, dtype=f32).reshape(1, -1, 1, 1)
    u = (u0[:, None] - (s * k).astype(f32)).astype(f32)
    return _rcp(u)


def _np32(x):
    if torch.is_tensor(x):
        return x.detach().cpu().numpy().astype(f32)
    return np.asarray(x, dtype=f32)


def ladder_f32(first, step, D, B, h, w):
    """The depths of an inverse ops.Ladder -> (B,D,h,w) float32, d_k = RN(1/RN(first - RN(step*k)))
    (inverse_plane, k1_common.cuh).  first: a float, a (B,) or a (B,h,w) array or tensor in
    1/depth; step: a float or a (B,) array or tensor."""
    fa, sa = _np32(first), _np32(step)
    u0 = fa.reshape(B, 1, h, w) if fa.ndim == 3 else np.broadcast_to(fa.reshape(-1, 1, 1, 1), (B, 1, 1, 1))
    s = np.broadcast_to(sa.reshape(-1, 1, 1, 1), (B, 1, 1, 1))
    k = np.arange(D, dtype=f32).reshape(1, -1, 1, 1)
    u = (u0 - (s * k).astype(f32)).astype(f32)
    return np.ascontiguousarray(np.broadcast_to(_rcp(u), (B, D, h, w)))


def regress_f64(logits, dv):
    """Rule 5 in float64: depth = 1 / sum_k p_k / d_k, with the uniform index and confidence."""
    lg = logits.double().cpu()
    d = dv.double().cpu()
    d = d.reshape(1, -1, 1, 1) if d.dim() == 1 else d
    p = torch.softmax(lg, 1)
    ubar = (p / d).sum(1)
    _, conf, index, _ = O.regress_depth(lg, d)
    return 1.0 / ubar, conf, index, p, ubar


def regress_bwd_f64(logits, dv, grad):
    """d depth / d logit_k = -depth^2 p_k (1/d_k - ubar) grad, float64."""
    depth, _, _, p, ubar = regress_f64(logits, dv)
    d = dv.double().cpu()
    d = d.reshape(1, -1, 1, 1) if d.dim() == 1 else d
    g = grad.double().cpu().unsqueeze(1)
    return -(depth ** 2).unsqueeze(1) * p * (1.0 / d - ubar.unsqueeze(1)) * g


def cascade_forward_inverse(sd, imgs, proj_mats, init_depth_min, depth_interval,
                            n_depths=(8, 32, 48), interval_ratios=(1, 2, 4), num_groups=1):
    """casmvs_oracle.cascade_forward with the inverse-depth sweep and regression, on CPU in the
    dtype of its inputs as cascade_forward runs.  The hypotheses follow rules 3-4 in float64 and
    are then rounded to that dtype."""
    B, V = imgs.shape[:2]
    H, W = imgs.shape[-2:]
    dt = imgs.dtype
    top = len(n_depths) - 1
    st = steps_f32(init_depth_min, depth_interval, n_depths, interval_ratios, B)
    un = torch.from_numpy(st[0].astype(np.float64))
    uf = torch.from_numpy(st[1].astype(np.float64))
    results = {}
    with torch.no_grad():
        feats = O.feature_pyramid(imgs.reshape(B * V, 3, H, W), sd)
        depth_l = None
        for l in range(top, -1, -1):
            f = feats[f"level_{l}"]
            f = f.reshape(B, V, *f.shape[1:])
            D = n_depths[l]
            h, w = f.shape[-2:]
            s = torch.from_numpy(st[2][l].astype(np.float64)).reshape(-1, 1, 1, 1)
            if l == top:
                u0 = un.reshape(-1, 1, 1, 1).expand(B, 1, h, w)
            else:
                c = O.upsample_depth(depth_l).double()
                u0 = torch.maximum(1.0 / c + D * 0.5 * s, uf.reshape(-1, 1, 1, 1) + (D - 1) * s)
            k = torch.arange(D, dtype=torch.float64).reshape(1, -1, 1, 1)
            dv = (1.0 / (u0 - s * k)).to(dt)
            if num_groups == 1:
                cost = O.variance_cost_volume(f, proj_mats[:, :, l], dv)
            else:
                cost = O.groupwise_cost_volume(f, proj_mats[:, :, l], dv, num_groups)
            logits = O.cost_regularize(cost, sd, f"cost_reg_{l}.").squeeze(1)
            p = F.softmax(logits, 1)
            depth_l = 1.0 / (p / dv).sum(1)
            _, conf_l, index_l, _ = O.regress_depth(logits, dv)
            results[f"depth_{l}"] = depth_l
            results[f"confidence_{l}"] = conf_l
            results[f"depth_index_{l}"] = index_l
    return results
