"""Float64 reference of the dynamic consistency fusion (geo_fuse_kernel<kDynamic>,
casmvs_geo_fuse_dynamic_fwd in csrc/fusion.cu) with admissible sets, for per-element checks.

Plain torch only (no casmvsnet_pl_b200 import).  The per-source path (projection, remap bins and
taps, back-projection) and its rounding bounds are those of oracle/fusion_fp64.py, whose helpers
this module calls; only the decision differs.  The rule:

* Source s is consistent at level k (k = 2..10) when e_pix < (k/4)^2 and e_dep < T_k =
  float32(k / 1300); k_s is its least such level, 0 for none (NaN compares false).
* n_k = #{s : 0 < k_s <= k}; the geometric mask holds when n_k >= k for some 2 <= k <= min(10, S).
* The average and geo_count take the sources with k_s > 0 (consistent at level 10).

Admissible levels.  Per remap candidate the kernel's fp32 e_pix lies within ep of the float64
p, and e_dep within et of t (fusion_fp64's bounds).  k_s is non-decreasing in both errors (0
counting as "above 10"), so it lies between the level of the lower corner (p - ep, t - et) and
that of the upper corner (p + ep, t + et); every level between is admissible.  The admissible
set of a (source, pixel) pair is the union of those intervals over the remap candidates, as a
bitmask (bit k for level k, bit 0 for "no level"); an unconstrained pair admits every level and
a reference depth that is 0 or not finite admits only 0.  Colour intervals and reprojection
bounds are taken over the candidates that admit consistency at level 10.

Everything downstream of the levels is checked from the kernel's own levels, which are checked
first: geo_count and the geometric mask exactly, mask_final with the confidence sets, and
depth_refined, image_refined and points with fusion_fp64's bounds.

``level_of`` and ``geometric_mask`` restate the rule on given errors, for known answers.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import fusion_fp64 as FF

LEVELS = tuple(range(2, 11))
PIX_DIV = 4
DEP_DIV = 1300
PIX_TH = {k: (k / PIX_DIV) ** 2 for k in LEVELS}                # k^2 / 16, exact in fp32
DEP_TH = {k: float(np.float32(k / DEP_DIV)) for k in LEVELS}    # rounded once from double
ALL_LEVELS = sum(1 << k for k in LEVELS) | 1
ORDER = ("level", "reproj", "geo_count", "mask_final", "depth_refined", "image_refined", "points")


# ------------------------------------------------------------------------------- the rule
def level_of(e_pix, e_dep):
    """Least level at which errors (e_pix, e_dep) are consistent, 0 for none (float64 or
    float32 arrays / tensors / scalars compared as given)."""
    e_pix, e_dep = torch.as_tensor(e_pix), torch.as_tensor(e_dep)
    out = torch.zeros(torch.broadcast_shapes(e_pix.shape, e_dep.shape), dtype=torch.int64)
    for k in reversed(LEVELS):
        out = torch.where((e_pix < PIX_TH[k]) & (e_dep < DEP_TH[k]), k, out)
    return out


def geometric_mask(levels):
    """levels (S, ...) -> the dynamic geometric mask (...): n_k >= k for some 2 <= k <= min(10, S)."""
    levels = torch.as_tensor(levels).long()
    S = levels.shape[0]
    keep = torch.zeros(levels.shape[1:], dtype=torch.bool, device=levels.device)
    for k in LEVELS:
        if k > S:
            break
        n_k = ((levels > 0) & (levels <= k)).sum(0)
        keep |= n_k >= k
    return keep


def _bits(lo, hi):
    """Bitmask of levels lo..hi (11 standing for 'no level', bit 0)."""
    out = torch.zeros_like(lo)
    for k in LEVELS:
        out |= torch.where((lo <= k) & (k <= hi), 1 << k, 0)
    return out | torch.where(hi == 11, 1, 0)


# ------------------------------------------------------------------------------- per source
@torch.no_grad()
def source_levels(depth_ref, depth_src, image_src, rs, sr, reproj=None, exact=False):
    """One source in float64 -> dict of (H, W) maps:
      sets           int64 bitmask of the admissible k_s (bit k for level k, bit 0 for 0),
      unconstrained  pairs where the projection is too close to a singularity,
      col_lo/col_hi  (H, W, 3) interval of the admissible colours of a source that joins the
                     average (None without images),
      rz_ratio       with ``reproj``: min over the candidates admitting level 10 of
                     |reproj - rz64| / e_rz (0 where equal, inf where none).
    The projection, bins, taps and bounds are fusion_fp64.source_ref's, step for step."""
    k = 0.0 if exact else 1.0
    ULP, SAFE, FLT_MAX = FF.ULP, FF.SAFE, FF.FLT_MAX
    dev = depth_ref.device
    d = depth_ref.double()
    H, W = d.shape
    y, x = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=dev),
                          torch.arange(W, dtype=torch.float64, device=dev), indexing="ij")
    A, B = FF._rows(rs), FF._rows(sr)
    X, Y = x * d, y * d
    ev = (ULP * X.abs(), ULP * Y.abs(), 0.0)
    qx, bx = FF._dot(A[0:4], (X, Y, d), ev, k)
    qy, by = FF._dot(A[4:8], (X, Y, d), ev, k)
    qz, bz = FF._dot(A[8:12], (X, Y, d), ev, k)
    bad_d = ~torch.isfinite(d) | (d == 0)
    xs, exs = FF._div(qx, bx, qz, bz, k)
    ys, eys = FF._div(qy, by, qz, bz, k)
    fin = torch.isfinite(xs) & torch.isfinite(ys)
    if exact:
        unc = torch.zeros_like(fin)
    else:
        unc = ~((qx.abs() + bx < FLT_MAX) & (qy.abs() + by < FLT_MAX) & (qz.abs() + bz < FLT_MAX)
                & (xs.abs() + exs < FLT_MAX) & (ys.abs() + eys < FLT_MAX))
    zero = torch.zeros_like(xs)
    tx, ty = torch.where(fin, 32 * xs, zero), torch.where(fin, 32 * ys, zero)
    etx, ety = torch.where(fin, 32 * exs, zero), torch.where(fin, 32 * eys, zero)
    lox, hix, offx, uncx = FF._bins(tx, etx, W)
    loy, hiy, offy, uncy = FF._bins(ty, ety, H)
    unc = (unc | ((uncx | uncy) & ~(offx | offy))) & ~bad_d

    dsrc = depth_src.double()
    isrc = image_src.double() if image_src is not None else None
    sets = torch.zeros(H, W, dtype=torch.int64, device=dev)
    inf = torch.full_like(xs, float("inf"))
    col_lo = inf.unsqueeze(-1).repeat(1, 1, 3) if isrc is not None else None
    col_hi = -col_lo if isrc is not None else None
    rz_ratio = inf.clone()
    for sx in (lox, hix):
        for sy in (loy, hiy):
            ds, eds = FF.remap_ref(dsrc, sx, sy, k)
            ds, eds = torch.where(fin, ds, zero), torch.where(fin, eds, zero)
            U, V = xs * ds, ys * ds
            EU = xs.abs() * eds + exs * (ds.abs() + eds)
            EV = ys.abs() * eds + eys * (ds.abs() + eds)
            eU = k * (EU + ULP * (U.abs() + EU)) * SAFE
            eV = k * (EV + ULP * (V.abs() + EV)) * SAFE
            evr = (eU, eV, eds)
            rx, brx = FF._dot(B[0:4], (U, V, ds), evr, k)
            ry, bry = FF._dot(B[4:8], (U, V, ds), evr, k)
            rz, brz = FF._dot(B[8:12], (U, V, ds), evr, k)
            rz_unc = (rz.abs() <= brz) if not exact else torch.zeros_like(fin)
            px, epx = FF._div(rx, brx, rz, brz, k)
            py, epy = FF._div(ry, bry, rz, brz, k)
            dx, dy = px - x, py - y
            edx = k * (epx + ULP * (dx.abs() + epx)) * SAFE
            edy = k * (epy + ULP * (dy.abs() + epy)) * SAFE
            p = dx * dx + dy * dy
            E = 2 * dx.abs() * edx + edx * edx + 2 * dy.abs() * edy + edy * edy
            ep = k * (E + 2 * ULP * (p + E)) * SAFE
            diff = rz - d
            tt = diff.abs() / d.abs()
            E = (brz + ULP * (diff.abs() + brz)) / d.abs()
            et = k * (E + ULP * (tt + E)) * SAFE
            lo = torch.full_like(sets, 11)             # least level admitted at the lower corner
            hi = torch.full_like(sets, 11)             # least level certain at the upper corner
            for lv in reversed(LEVELS):
                can = ((p - ep < PIX_TH[lv]) | rz_unc) & (tt - et < DEP_TH[lv]) & ~bad_d
                sure = (p + ep < PIX_TH[lv]) & ~rz_unc & (tt + et < DEP_TH[lv]) & ~bad_d
                lo = torch.where(can, lv, lo)
                hi = torch.where(sure, lv, hi)
            sets |= _bits(lo, hi)
            c_t = lo <= LEVELS[-1]                     # this candidate may join the average
            if isrc is not None:
                col, ecol = FF.remap_ref(isrc, sx, sy, k)
                m3 = (c_t & fin).unsqueeze(-1)
                col_lo = torch.where(m3, torch.minimum(col_lo, col - ecol), col_lo)
                col_hi = torch.where(m3, torch.maximum(col_hi, col + ecol), col_hi)
                z3 = (c_t & ~fin).unsqueeze(-1)        # remap skipped: colour 0 exactly
                col_lo = torch.where(z3, torch.minimum(col_lo, torch.zeros_like(col_lo)), col_lo)
                col_hi = torch.where(z3, torch.maximum(col_hi, torch.zeros_like(col_hi)), col_hi)
            if reproj is not None:
                r = reproj.double()
                q = (r - rz).abs() / brz
                q = torch.where(r == rz, zero, torch.nan_to_num(q, nan=float("inf")))
                rz_ratio = torch.where(c_t, torch.minimum(rz_ratio, q), rz_ratio)
    sets = torch.where(unc, ALL_LEVELS, sets)
    if isrc is not None:
        u3 = unc.unsqueeze(-1)
        col_lo = torch.where(u3, -torch.ones_like(col_lo) * float("inf"), col_lo)
        col_hi = torch.where(u3, torch.ones_like(col_hi) * float("inf"), col_hi)
    rz_ratio = torch.where(unc, zero, rz_ratio)
    return dict(sets=sets, unconstrained=unc, col_lo=col_lo, col_hi=col_hi, rz_ratio=rz_ratio)


def _popcount(v):
    n = torch.zeros_like(v)
    for b in range(11):
        n += (v >> b) & 1
    return n


class DynamicReport(FF.FuseReport):
    """FuseReport with the per-source quantity named 'level'; ambiguous counts the (source,
    pixel) pairs with more than one admissible level."""

    def first_failure(self):
        for name in ORDER:
            if name in self.q and self.q[name]["bad"]:
                return name, self.q[name]["first"]
        return None

    def describe(self):
        parts = []
        for name in ORDER:
            if name in self.q:
                e = self.q[name]
                parts.append(f"{name}: {e['bad']} bad, worst ratio {e['worst']:.3g}"
                             + (f", first at {e['first']}" if e["first"] is not None else ""))
        return ("; ".join(parts) + f"; ambiguous {self.ambiguous} of {self.pairs} pairs "
                f"({self.unconstrained} unconstrained), certain level {self.certain_true}, "
                f"certain none {self.certain_false}, confidence ambiguous {self.conf_ambiguous}")


@torch.no_grad()
def check_fuse_dynamic(inp, out, exact=False, device=None):
    """Every output of one casmvs_geo_fuse_dynamic_fwd call against float64 applied to its own
    inputs (fusion_fp64.check_fuse's inputs; min_consistent is not used).
    out: level (S, H, W) uint8, reproj (S, H, W), geo_count, mask_final (bool), depth_refined,
    image_refined | None, points | None.  With ``exact`` only level, reproj, geo_count and
    mask_final are checked, against the rounding-free outcome."""
    dev = device or inp["depth_ref"].device

    def t(v):
        return None if v is None else torch.as_tensor(v).to(dev)
    d32 = t(inp["depth_ref"])
    H, W = d32.shape
    S = len(inp["depth_srcs"])
    rs = np.asarray(inp["rs"], np.float32).reshape(-1, 12)
    sr = np.asarray(inp["sr"], np.float32).reshape(-1, 12)
    img_ref = t(inp.get("image_ref"))
    img_srcs = inp.get("image_srcs")
    use_img = img_ref is not None and img_srcs is not None
    level, reproj = t(out["level"]).long(), t(out["reproj"])
    rep = DynamicReport()
    lo = img_ref.double().clone() if img_ref is not None else None
    hi = lo.clone() if lo is not None else None
    amag = lo.abs() if lo is not None else None
    for s in range(S):
        sref = source_levels(d32, t(inp["depth_srcs"][s]), t(img_srcs[s]) if use_img else None,
                             rs[s], sr[s], reproj=reproj[s], exact=exact)
        sets, lv = sref["sets"], level[s]
        n = _popcount(sets)
        rep.pairs += H * W
        rep.ambiguous += int((n > 1).sum())
        rep.unconstrained += int(sref["unconstrained"].sum())
        rep.certain_true += int(((n == 1) & (sets != 1)).sum())
        rep.certain_false += int((sets == 1).sum())
        ok = (lv >= 0) & (lv <= LEVELS[-1]) & (lv != 1) & (((sets >> lv.clamp(0, 62)) & 1) == 1)
        rep.add("level", ~ok, prefix=(s,))
        m = lv > 0
        r = sref["rz_ratio"]
        rep.add("reproj", (m & ~(r <= 1)) | (~m & (reproj[s] != 0)), r, m, prefix=(s,))
        if lo is not None and use_img:
            m3 = m.unsqueeze(-1)
            lo = lo + torch.where(m3, sref["col_lo"], torch.zeros_like(lo))
            hi = hi + torch.where(m3, sref["col_hi"], torch.zeros_like(hi))
            amag = amag + torch.where(m3, torch.maximum(sref["col_lo"].abs(), sref["col_hi"].abs()),
                                      torch.zeros_like(amag))
    mask = level > 0
    cnt = t(out["geo_count"]).long()
    rep.add("geo_count", cnt != mask.long().sum(0))

    keep = geometric_mask(level) if S else torch.zeros(H, W, dtype=torch.bool, device=dev)
    mf = t(out["mask_final"]).bool()
    if inp.get("proba_ref") is not None:
        up, e = FF.upsample4_ref(t(inp["proba_ref"]))
        c32 = FF.f32(inp["conf"])
        can_t, can_f = up + e > c32, ~(up - e > c32)
        rep.conf_ambiguous = int((can_t & can_f).sum())
        rep.add("mask_final", (mf & ~(keep & can_t)) | (~mf & keep & ~can_f))
    else:
        rep.add("mask_final", mf != keep)
    if exact:
        return rep

    # the averages and the points from the kernel's own levels, geo_count and reprojections:
    # fusion_fp64.check_fuse's bounds
    ULP, SAFE, F64 = FF.ULP, FF.SAFE, FF.F64
    n1 = (cnt + 1).double()
    d = d32.double()
    R = reproj.double() * mask
    dsum = d + R.sum(0)
    Am = d.abs() + R.abs().sum(0)
    want = dsum / n1
    b = (cnt.double() * ULP * Am * SAFE) / n1
    b = (b + ULP * (want.abs() + b)) * SAFE + F64 * Am
    got = t(out["depth_refined"]).double()
    q = (got - want).abs() / b
    q = torch.where(got == want, torch.zeros_like(q), torch.nan_to_num(q, nan=float("inf")))
    q = torch.where(torch.isnan(got) & torch.isnan(want), torch.zeros_like(q), q)
    rep.add("depth_refined", ~(q <= 1), q)

    if out.get("image_refined") is not None and lo is not None:
        inv = (1.0 / n1).unsqueeze(-1)
        c3 = cnt.double().unsqueeze(-1)
        b = (c3 * ULP * amag + 2 * ULP * amag * (1 + c3 * ULP)) * inv * SAFE + F64 * amag
        got = t(out["image_refined"]).double()
        q = FF._ratio_outside(got, lo * inv, hi * inv, b)
        rep.add("image_refined", ~(q <= 1), q)

    if out.get("points") is not None:
        M = FF._rows(inp["ref2world"])
        dref = t(out["depth_refined"]).double()
        y, x = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=dev),
                              torch.arange(W, dtype=torch.float64, device=dev), indexing="ij")
        X, Y = x * dref, y * dref
        ev = (ULP * X.abs(), ULP * Y.abs(), 0.0)
        got = t(out["points"]).double()
        qs = []
        for r in range(3):
            v, bv = FF._dot(M[4 * r:4 * r + 4], (X, Y, dref), ev, 1.0)
            g = got[..., r]
            qr = (g - v).abs() / bv
            qr = torch.where(g == v, torch.zeros_like(qr), torch.nan_to_num(qr, nan=float("inf")))
            qr = torch.where(torch.isnan(g) & torch.isnan(v), torch.zeros_like(qr), qr)
            qs.append(qr)
        rep.add("points", ~(torch.stack(qs, -1) <= 1), torch.stack(qs, -1))
    return rep


# ------------------------------------------------------------------------------- known answers
def edge_cases(seed=0):
    """fusion_fp64.edge_cases (their fp32 arithmetic is exact or far from every threshold, so
    ``exact=True`` states the kernel's outcome at every level too) plus:

    levels        constant depth 512 seen through pure shifts whose pixel errors sit exactly on
                  the level thresholds (k/4 px: not consistent at k, so level k + 1) and between
                  them, so that the sources' levels are 2..10 and 0 and n_k crosses k at several
                  pixels of a depth step.
    """
    out = list(FF.edge_cases(seed))
    rng = np.random.default_rng(seed + 1)
    H, W = 12, 16
    d512 = np.full((H, W), 512, np.float32)
    # back shifts leave dx = a - b: exactly k/4 (level k + 1), or k/4 - 1/8 (level k)
    errs = [0.125, 0.375, 0.5, 0.625, 0.875, 1.0, 1.375, 2.25, 2.5, 3.0]
    rows = [(FF.shift_rows(2.0, 0), FF.shift_rows(-2.0 + e, 0)) for e in errs]
    out.append(("levels", FF._inputs(d512, [d512] * len(rows), rows, rng)))
    return out
