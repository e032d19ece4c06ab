"""Float64 reference of the geometric-consistency fusion kernel (geo_fuse_kernel,
csrc/fusion.cu) with admissible sets, for per-element checks.

Plain torch only (no casmvsnet_pl_b200 import), on the CPU or the GPU.  The inputs are exactly
what casmvs_geo_fuse_fwd receives: the float32 depth / image / proba maps of the reference view,
the float32 depth maps and images of the sources, the float32 3x4 rows proj_ref2src (``rs``) and
proj_src2ref (``sr``), ref2world (4x4), conf and min_consistent.

Every outcome of one (source s, pixel) pair hangs on discrete fp32 decisions: the remap bin
rint(32 x), dx^2 + dy^2 < 1, |rz - d| / d < 0.01f, and up(proba) > conf.  A tolerance cannot
describe how those differ from float64, so the reference returns the set of admissible outcomes.
u = 2^-24, SAFE = 1 + 2^-20 covers second-order terms.  Each bound holds whether or not nvcc
contracts a product and a sum into an FMA (an FMA only removes roundings), and whatever the order
of the four-term sums (any order of a length-n dot product is within gamma_n of it):

* Projection.  X = fl(x d), Y = fl(y d) are each within u |x d| of x d (x, y are exact
  integers).  qx = A0 X + A1 Y + A2 d + A3 (likewise qy, qz) is a four-term dot product:
      |qx32 - qx64| <= 4u M + u (|A0 x d| + |A1 y d|),   M = sum_k |A_k| |v_k|,  v = (X, Y, d, 1).
  xs = fl(qx / qz): with e_x, e_z the bounds above,
      E = (e_x + |xs64| e_z) / (|qz64| - e_z),   |xs32 - xs64| <= E + u (|xs64| + E).
  Where |qz64| <= e_z (or qx, qz or xs may leave the float range) the pair is unconstrained:
  mask True and False are both admissible, and so is any reprojection and colour.
* Bins.  The kernel rounds 32 xs32 (exact) half to even and saturates to int32.  Per axis the
  candidates are every integer between rint(32 (xs64 - e)) and rint(32 (xs64 + e)) (rint is
  monotone): one bin, or two where the interval holds a half-integer.  More than two makes the
  pair unconstrained, unless every candidate bin puts both taps of that axis off the image (then
  the remap reads 0 whichever it is).  Up to 4 (sx, sy) candidates.
* Remap, per candidate.  ix = sx >> 5, fx = (sx & 31) / 32; the four weights are exact in fp32
  (products of multiples of 1/32); taps off the image read 0.  The kernel rounds the four
  products and three sums: |ds32 - ds64| <= 4u sum_k |t_k| w_k, and 0 when fx = fy = 0 (one
  weight 1, the others 0).  Colours the same per channel.  A NaN tap makes ds NaN in both, even
  at weight 0 (NaN * 0).
* Reprojection.  U = fl(xs32 ds32) uses the kernel's own fp32 xs, not the bin centre:
      E = |xs64| e_ds + e_xs (|ds64| + e_ds),   |U32 - xs64 ds64| <= E + u (|U64| + E).
  rx, ry, rz are four-term dot products of sr with (U, V, ds, 1) whose inputs carry e_U, e_V,
  e_ds:  e_r = (|B0| e_U + |B1| e_V + |B2| e_ds)(1 + 4u) + 4u M_r.
* Pixel test.  px = fl(rx / rz) as for xs (|rz64| <= e_rz: either outcome); dx = fl(px - x)
  adds u (|dx| + e_px); p = dx^2 + dy^2 (two products and a sum, or an FMA):
      e_p = (sum 2|dx| e_dx + e_dx^2) + 2u (p64 + that).
  True is admissible where p64 - e_p < 1, False where p64 + e_p >= 1.
* Depth test.  t = |fl(fl(rz - d) / d)|: e_t = E + u (t64 + E), E = (e_rz + u (|rz64 - d| +
  e_rz)) / |d|, against 0.01f.  The reference's eval.py states 0.01; float64 0.01 differs from
  0.01f by 2e-10 relative (2.2e-12 absolute at t = 0.01), inside every margin bound
  (e_t >= u t = 6e-10 there).  A depth d that is 0 or not finite fails the test in the kernel
  ((rz - d) / d is inf or NaN), so its mask is False for certain.
* Mask.  Per candidate the mask is pixel-test AND depth-test; the admissible set per (s, pixel)
  is the union over the candidates: {True}, {False} or {True, False}.  A True mask must carry a
  reprojection within e_rz of the rz64 of a candidate that admits True, and a colour within the
  colour bound of one.
* Confidence.  cv2.resize(proba, fx=4, INTER_LINEAR): source coordinate (x + 0.5) / 4 - 0.5,
  replicated border, fractions in {0, 1/8, 3/8, 5/8, 7/8} exact.  The kernel blends a row
  (2 products, 1 sum: 2u of the weighted magnitudes, 0 when fx = 0) and then the two rows
  (again 2u, 0 when fy = 0).  The decision up > float32(conf) is certain where up64 is farther
  than that bound from float32(conf); at the 2x2 corner blocks the bound is 0, so a proba of
  exactly float32(conf) is rejected there and the next float above accepted.
* Refinement.  depth_refined = fl((d + sum_s reproj_s) / (cnt + 1)), a sequential fp32 sum of
  cnt + 1 terms (cnt u sum |terms|) and a division (u); the check takes the kernel's own
  reproj and geo_count, which are checked first, so errors do not compound.  image_refined =
  (image_ref + sum_s col_s) * fl(1 / (cnt + 1)): it must lie in the interval sum of the
  admissible colours, widened by the sum's cnt u A and 2u A for the reciprocal and the product.
  points = ref2world . (fl(x dref), fl(y dref), dref, 1) with the kernel's own dref: a projection
  bound as above.

``exact=True`` sets every rounding bound of the per-source path to 0.  It gives the kernel's
outcome only for inputs whose fp32 arithmetic is exact or far from every threshold by
construction (the known-answer cases of ``edge_cases``): pure pixel shifts with power-of-two
depths, where xs lands exactly on 1/64-px ties and dx^2 + dy^2 can be exactly 1.
"""
from __future__ import annotations

import numpy as np
import torch

ULP = 2.0 ** -24
SAFE = 1 + 2.0 ** -20
F64 = 2.0 ** -50                     # the oracle's own float64 rounding, relative to magnitudes
MAX_SRC = 16
DEP_TH = float(np.float32(0.01))     # the kernel's 0.01f
FLT_MAX = float(np.finfo(np.float32).max)
INT_MIN, INT_MAX = -2.0 ** 31, 2.0 ** 31 - 1
ORDER = ("mask", "reproj", "geo_count", "mask_final", "depth_refined", "image_refined", "points")


def f32(v):
    """The float32 value a Python float becomes at the C boundary (ctypes c_float)."""
    return float(np.float32(v))


def _rows(M):
    return [float(v) for v in np.asarray(M, dtype=np.float32).reshape(-1)]


def _dot(a, v, ev, k):
    """a[0] v0 + a[1] v1 + a[2] v2 + a[3] in float64 -> value, bound (inputs carry ev)."""
    val = a[0] * v[0] + a[1] * v[1] + a[2] * v[2] + a[3]
    mag = abs(a[0]) * v[0].abs() + abs(a[1]) * v[1].abs() + abs(a[2]) * v[2].abs() + abs(a[3])
    inp = abs(a[0]) * ev[0] + abs(a[1]) * ev[1] + abs(a[2]) * ev[2]
    return val, k * ((inp * (1 + 4 * ULP) + 4 * ULP * mag) * SAFE + F64 * mag)


def _div(num, en, den, ed, k):
    """fl(num / den) with inputs within en, ed -> value, bound (inf where den may be 0)."""
    q = num / den
    room = den.abs() - ed
    E = (en + q.abs() * ed) / room
    b = (E + ULP * (q.abs() + E)) * SAFE
    b = torch.where(room > 0, b, torch.full_like(b, float("inf")))
    return q, k * b if k else torch.zeros_like(q)


def _bins(t, et, n):
    """Candidate bins of one axis: lo, hi (int64), all taps off the image, unconstrained."""
    lo = torch.round(t - et).clamp(INT_MIN, INT_MAX)
    hi = torch.round(t + et).clamp(INT_MIN, INT_MAX)
    off = (lo >= 32 * n) | (hi <= -33)
    return lo.long(), hi.long(), off, (hi - lo > 1) & ~off


def _taps(img, ix, iy):
    H, W = img.shape[:2]
    ok = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
    v = img[iy.clamp(0, H - 1), ix.clamp(0, W - 1)]
    if img.dim() == 3:
        ok = ok.unsqueeze(-1)
    return torch.where(ok, v, torch.zeros_like(v))


def remap_ref(img, sx, sy, k=1):
    """cv2.remap INTER_LINEAR of a float64 map at integer 1/32-px positions -> value, bound."""
    ix, iy = torch.div(sx, 32, rounding_mode="floor"), torch.div(sy, 32, rounding_mode="floor")
    fx, fy = (sx - 32 * ix).double() / 32, (sy - 32 * iy).double() / 32
    w = ((1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy)
    exact = (fx == 0) & (fy == 0)
    if img.dim() == 3:
        w = tuple(v.unsqueeze(-1) for v in w)
        exact = exact.unsqueeze(-1)
    t = (_taps(img, ix, iy), _taps(img, ix + 1, iy), _taps(img, ix, iy + 1), _taps(img, ix + 1, iy + 1))
    val = t[0] * w[0] + t[1] * w[1] + t[2] * w[2] + t[3] * w[3]
    mag = sum(tk.abs() * wk for tk, wk in zip(t, w))
    b = torch.where(exact, torch.zeros_like(mag), (4 * ULP * mag) * SAFE + F64 * mag)
    return val, k * b


@torch.no_grad()
def source_ref(depth_ref, depth_src, image_src, rs, sr, reproj=None, exact=False):
    """One source of geo_fuse_kernel in float64 -> dict of (H, W) maps:
      can_true, can_false   the admissible mask set,
      unconstrained         pairs where the projection is too close to a singularity,
      col_lo, col_hi        (H, W, 3) interval of the admissible colours (None without images),
      rz_ratio              with ``reproj``: min over the candidates admitting True of
                            |reproj - rz64| / e_rz (0 where equal, inf where none).
    rs, sr: the 12 float32 values of the 3x4 rows the kernel receives."""
    k = 0.0 if exact else 1.0
    dev = depth_ref.device
    d = depth_ref.double()
    H, W = d.shape
    y, x = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=dev),
                          torch.arange(W, dtype=torch.float64, device=dev), indexing="ij")
    A, B = _rows(rs), _rows(sr)
    X, Y = x * d, y * d
    ev = (ULP * X.abs(), ULP * Y.abs(), 0.0)
    qx, bx = _dot(A[0:4], (X, Y, d), ev, k)
    qy, by = _dot(A[4:8], (X, Y, d), ev, k)
    qz, bz = _dot(A[8:12], (X, Y, d), ev, k)
    bad_d = ~torch.isfinite(d) | (d == 0)
    xs, exs = _div(qx, bx, qz, bz, k)
    ys, eys = _div(qy, by, qz, bz, k)
    fin = torch.isfinite(xs) & torch.isfinite(ys)
    if exact:
        unc = torch.zeros_like(fin)
    else:
        unc = ~((qx.abs() + bx < FLT_MAX) & (qy.abs() + by < FLT_MAX) & (qz.abs() + bz < FLT_MAX)
                & (xs.abs() + exs < FLT_MAX) & (ys.abs() + eys < FLT_MAX))
    zero = torch.zeros_like(xs)
    tx, ty = torch.where(fin, 32 * xs, zero), torch.where(fin, 32 * ys, zero)
    etx, ety = torch.where(fin, 32 * exs, zero), torch.where(fin, 32 * eys, zero)
    lox, hix, offx, uncx = _bins(tx, etx, W)
    loy, hiy, offy, uncy = _bins(ty, ety, H)
    unc = (unc | ((uncx | uncy) & ~(offx | offy))) & ~bad_d

    dsrc = depth_src.double()
    isrc = image_src.double() if image_src is not None else None
    ct = torch.zeros_like(fin)
    cf = torch.zeros_like(fin)
    inf = torch.full_like(xs, float("inf"))
    col_lo = inf.unsqueeze(-1).repeat(1, 1, 3) if isrc is not None else None
    col_hi = -col_lo if isrc is not None else None
    rz_ratio = inf.clone()
    for sx in (lox, hix):
        for sy in (loy, hiy):
            ds, eds = remap_ref(dsrc, sx, sy, k)
            ds, eds = torch.where(fin, ds, zero), torch.where(fin, eds, zero)
            U, V = xs * ds, ys * ds                    # xs * 0 is NaN where xs is not finite
            EU = xs.abs() * eds + exs * (ds.abs() + eds)
            EV = ys.abs() * eds + eys * (ds.abs() + eds)
            eU = k * (EU + ULP * (U.abs() + EU)) * SAFE
            eV = k * (EV + ULP * (V.abs() + EV)) * SAFE
            evr = (eU, eV, eds)
            rx, brx = _dot(B[0:4], (U, V, ds), evr, k)
            ry, bry = _dot(B[4:8], (U, V, ds), evr, k)
            rz, brz = _dot(B[8:12], (U, V, ds), evr, k)
            rz_unc = (rz.abs() <= brz) if not exact else torch.zeros_like(fin)
            px, epx = _div(rx, brx, rz, brz, k)
            py, epy = _div(ry, bry, rz, brz, k)
            dx, dy = px - x, py - y
            edx = k * (epx + ULP * (dx.abs() + epx)) * SAFE
            edy = k * (epy + ULP * (dy.abs() + epy)) * SAFE
            p = dx * dx + dy * dy
            E = 2 * dx.abs() * edx + edx * edx + 2 * dy.abs() * edy + edy * edy
            ep = k * (E + 2 * ULP * (p + E)) * SAFE
            ct_pix = (p - ep < 1) | rz_unc
            cf_pix = ~(p + ep < 1) | rz_unc
            diff = rz - d
            tt = diff.abs() / d.abs()
            E = (brz + ULP * (diff.abs() + brz)) / d.abs()
            et = k * (E + ULP * (tt + E)) * SAFE
            c_t = ct_pix & (tt - et < DEP_TH) & ~bad_d
            c_f = cf_pix | ~(tt + et < DEP_TH) | bad_d
            ct |= c_t
            cf |= c_f
            if isrc is not None:
                col, ecol = remap_ref(isrc, sx, sy, k)
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
    ct |= unc
    cf |= unc
    if isrc is not None:
        u3 = unc.unsqueeze(-1)
        col_lo = torch.where(u3, -torch.ones_like(col_lo) * float("inf"), col_lo)
        col_hi = torch.where(u3, torch.ones_like(col_hi) * float("inf"), col_hi)
    rz_ratio = torch.where(unc, zero, rz_ratio)
    return dict(can_true=ct, can_false=cf, unconstrained=unc, col_lo=col_lo, col_hi=col_hi,
                rz_ratio=rz_ratio)


@torch.no_grad()
def upsample4_ref(proba):
    """cv2.resize(proba, fx=4, fy=4, INTER_LINEAR) in float64 -> value, bound of the kernel's
    fp32 blend (0 where both fractions are 0)."""
    p = proba.double()
    h4, w4 = p.shape
    dev = p.device

    def coords(n_out, n_in):
        f = (torch.arange(n_out, dtype=torch.float64, device=dev) + 0.5) * 0.25 - 0.5
        s = torch.floor(f)
        f = f - s
        lo, hi = s < 0, s >= n_in - 1
        f = torch.where(lo | hi, torch.zeros_like(f), f)
        s = torch.where(lo, torch.zeros_like(s), torch.where(hi, torch.full_like(s, n_in - 1), s)).long()
        return s, (s + 1).clamp(max=n_in - 1), f
    x0, x1, fx = coords(4 * w4, w4)
    y0, y1, fy = coords(4 * h4, h4)
    fx, fy = fx.view(1, -1), fy.view(-1, 1)

    def row(yy):
        a, b = p[yy][:, x0], p[yy][:, x1]
        v = a * (1 - fx) + b * fx
        m = a.abs() * (1 - fx) + b.abs() * fx
        return v, torch.where(fx == 0, torch.zeros_like(m), 2 * ULP * m)
    r0, e0 = row(y0)
    r1, e1 = row(y1)
    up = r0 * (1 - fy) + r1 * fy
    m = (r0.abs() + e0) * (1 - fy) + (r1.abs() + e1) * fy
    e = (1 - fy) * e0 + fy * e1 + torch.where(fy == 0, torch.zeros_like(m), 2 * ULP * m)
    return up, e * SAFE


class FuseReport:
    """Per quantity: number of failing elements, worst err/bound ratio and the first failure,
    as (s, y, x) for the per-source outputs and (y, x) for the others."""

    def __init__(self):
        self.q = {}
        self.ambiguous = 0          # (s, pixel) pairs with both mask values admissible
        self.unconstrained = 0
        self.conf_ambiguous = 0
        self.certain_true = 0
        self.certain_false = 0
        self.pairs = 0

    def add(self, name, bad, ratio=None, where=None, prefix=()):
        e = self.q.setdefault(name, dict(bad=0, worst=0.0, first=None))
        if bad.dim() == 3 and not prefix:
            bad = bad.any(-1)
        nb = int(bad.sum())
        e["bad"] += nb
        if nb and e["first"] is None:
            e["first"] = prefix + tuple(int(v) for v in bad.nonzero()[0][:2])
        if ratio is not None:
            r = ratio[where] if where is not None else ratio.reshape(-1)
            if r.numel():
                r = torch.nan_to_num(r.double(), nan=float("inf"))
                e["worst"] = max(e["worst"], float(r.max()))

    @property
    def ok(self):
        return all(e["bad"] == 0 for e in self.q.values())

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
                f"({self.unconstrained} unconstrained), certain True {self.certain_true}, "
                f"certain False {self.certain_false}, confidence ambiguous {self.conf_ambiguous}")


def _ratio_outside(got, lo, hi, b):
    """Distance of got outside [lo, hi] over b (0 inside, inf where b = 0 and outside)."""
    dist = torch.clamp(lo - got, min=0) + torch.clamp(got - hi, min=0)
    q = dist / b
    return torch.where(dist == 0, torch.zeros_like(q), torch.nan_to_num(q, nan=float("inf")))


@torch.no_grad()
def check_fuse(inp, out, exact=False, device=None):
    """Every output of one casmvs_geo_fuse_fwd call against float64 applied to its own inputs.

    inp: depth_ref, image_ref | None, proba_ref | None, depth_srcs [S], image_srcs [S] | None,
    rs, sr (S, 12) float32, ref2world (4, 4) float32, conf, min_consistent.
    out: mask (S, H, W) bool, reproj (S, H, W), geo_count, mask_final (bool), depth_refined,
    image_refined | None, points | None.  With ``exact`` only the mask, reproj, geo_count and
    mask_final are checked, against the rounding-free outcome (see the module docstring)."""
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
    mask, reproj = t(out["mask"]).bool(), t(out["reproj"])
    rep = FuseReport()
    msum = torch.zeros(H, W, dtype=torch.int64, device=dev)
    lo = img_ref.double().clone() if img_ref is not None else None
    hi = lo.clone() if lo is not None else None
    amag = lo.abs() if lo is not None else None
    for s in range(S):
        sref = source_ref(d32, t(inp["depth_srcs"][s]), t(img_srcs[s]) if use_img else None,
                          rs[s], sr[s], reproj=reproj[s], exact=exact)
        ct, cf, m = sref["can_true"], sref["can_false"], mask[s]
        rep.pairs += H * W
        rep.ambiguous += int((ct & cf).sum())
        rep.unconstrained += int(sref["unconstrained"].sum())
        rep.certain_true += int((ct & ~cf).sum())
        rep.certain_false += int((cf & ~ct).sum())
        rep.add("mask", (m & ~ct) | (~m & ~cf), prefix=(s,))
        r = sref["rz_ratio"]
        rep.add("reproj", (m & ~(r <= 1)) | (~m & (reproj[s] != 0)), r, m, prefix=(s,))
        msum += m.long()
        if lo is not None and use_img:
            m3 = m.unsqueeze(-1)
            lo = lo + torch.where(m3, sref["col_lo"], torch.zeros_like(lo))
            hi = hi + torch.where(m3, sref["col_hi"], torch.zeros_like(hi))
            amag = amag + torch.where(m3, torch.maximum(sref["col_lo"].abs(), sref["col_hi"].abs()),
                                      torch.zeros_like(amag))
    cnt = t(out["geo_count"]).long()
    rep.add("geo_count", cnt != msum)

    keep = cnt >= int(inp["min_consistent"])
    mf = t(out["mask_final"]).bool()
    if inp.get("proba_ref") is not None:
        up, e = upsample4_ref(t(inp["proba_ref"]))
        c32 = f32(inp["conf"])
        can_t, can_f = up + e > c32, ~(up - e > c32)     # admissible confidence outcomes
        rep.conf_ambiguous = int((can_t & can_f).sum())
        rep.add("mask_final", (mf & ~(keep & can_t)) | (~mf & keep & ~can_f))
    else:
        rep.add("mask_final", mf != keep)
    if exact:
        return rep

    n1 = (cnt + 1).double()
    d = d32.double()
    R = reproj.double() * mask
    dsum = d + R.sum(0)
    A = d.abs() + R.abs().sum(0)
    want = dsum / n1
    b = (cnt.double() * ULP * A * SAFE) / n1
    b = (b + ULP * (want.abs() + b)) * SAFE + F64 * A
    got = t(out["depth_refined"]).double()
    q = (got - want).abs() / b
    q = torch.where(got == want, torch.zeros_like(q), torch.nan_to_num(q, nan=float("inf")))
    both_nan = torch.isnan(got) & torch.isnan(want)
    q = torch.where(both_nan, torch.zeros_like(q), q)
    rep.add("depth_refined", ~(q <= 1), q)

    if out.get("image_refined") is not None and lo is not None:
        inv = (1.0 / n1).unsqueeze(-1)
        b = (cnt.double().unsqueeze(-1) * ULP * amag + 2 * ULP * amag * (1 + cnt.double().unsqueeze(-1) * ULP)) * inv * SAFE
        b = b + F64 * amag
        got = t(out["image_refined"]).double()
        q = _ratio_outside(got, lo * inv, hi * inv, b)
        rep.add("image_refined", ~(q <= 1), q)

    if out.get("points") is not None:
        M = _rows(inp["ref2world"])
        dref = t(out["depth_refined"]).double()
        y, x = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=dev),
                              torch.arange(W, dtype=torch.float64, device=dev), indexing="ij")
        X, Y = x * dref, y * dref
        ev = (ULP * X.abs(), ULP * Y.abs(), 0.0)
        got = t(out["points"]).double()
        qs = []
        for r in range(3):
            v, bv = _dot(M[4 * r:4 * r + 4], (X, Y, dref), ev, 1.0)
            g = got[..., r]
            qr = (g - v).abs() / bv
            qr = torch.where(g == v, torch.zeros_like(qr), torch.nan_to_num(qr, nan=float("inf")))
            qr = torch.where(torch.isnan(g) & torch.isnan(v), torch.zeros_like(qr), qr)
            qs.append(qr)
        q = torch.stack(qs, -1)
        rep.add("points", ~(q <= 1), q)
    return rep


# ------------------------------------------------------------------------------- scenes
def rel(P_a, P_b):
    """(P_a @ inv(P_b))[:3] in float32 numpy, as fusion.refine_ref_view passes it (eval.py:120)."""
    P_a, P_b = np.asarray(P_a, np.float32), np.asarray(P_b, np.float32)
    return np.ascontiguousarray((P_a @ np.ascontiguousarray(np.linalg.inv(P_b)))[:3], np.float32)


def scene_inputs(views, S, seed=0, noise=0.004, proba=True, conf=0.9, min_consistent=3):
    """Fusion inputs from rendered views (dicts of depth, P): view 0 is the reference, views
    1..S its sources.  Depths get seeded multiplicative noise (so many pairs sit near the 1 %
    depth test), images are random 0..255 integers, proba (H/4, W/4) is uniform in
    [conf - 0.1, 1].  Adds P_ref and P_srcs for fusion.refine_ref_view."""
    g = torch.Generator().manual_seed(seed)
    rng = np.random.default_rng(seed)
    H, W = views[0]["depth"].shape

    def depth(v):
        dd = v["depth"].detach().cpu().float()
        return (dd * (1 + noise * torch.randn(dd.shape, generator=g))).float()

    def image():
        return torch.from_numpy(rng.integers(0, 256, (H, W, 3)).astype(np.float32))
    P = [np.asarray(v["P"], np.float32) for v in views[:S + 1]]
    pr = None
    if proba:
        pr = torch.from_numpy(rng.uniform(conf - 0.1, 1.0, (H // 4, W // 4)).astype(np.float32))
    return dict(depth_ref=depth(views[0]), image_ref=image(), proba_ref=pr,
                depth_srcs=[depth(v) for v in views[1:S + 1]], image_srcs=[image() for _ in range(S)],
                rs=np.stack([rel(Ps, P[0]) for Ps in P[1:]]).reshape(S, 12) if S else np.zeros((0, 12), np.float32),
                sr=np.stack([rel(P[0], Ps) for Ps in P[1:]]).reshape(S, 12) if S else np.zeros((0, 12), np.float32),
                ref2world=np.ascontiguousarray(np.linalg.inv(P[0]), np.float32),
                conf=conf, min_consistent=min_consistent, P_ref=P[0], P_srcs=P[1:])


# ------------------------------------------------------------------------------- known answers
def shift_rows(a, b):
    """3x4 rows of a pure pixel shift: (x, y, d) -> (x + a, y + b) at depth d (float32)."""
    return np.array([[1, 0, a, 0], [0, 1, b, 0], [0, 0, 1, 0]], np.float32).reshape(-1)


def _inputs(d_ref, srcs, rows, rng, proba=None, conf=0.999, min_consistent=1):
    H, W = d_ref.shape
    img = lambda: torch.from_numpy(rng.integers(0, 256, (H, W, 3)).astype(np.float32))
    return dict(depth_ref=torch.from_numpy(np.ascontiguousarray(d_ref, np.float32)),
                image_ref=img(),
                proba_ref=None if proba is None else torch.from_numpy(np.ascontiguousarray(proba, np.float32)),
                depth_srcs=[torch.from_numpy(np.ascontiguousarray(s, np.float32)) for s in srcs],
                image_srcs=[img() for _ in srcs],
                rs=np.stack([r[0] for r in rows]) if rows else np.zeros((0, 12), np.float32),
                sr=np.stack([r[1] for r in rows]) if rows else np.zeros((0, 12), np.float32),
                ref2world=np.array([[1, 0, 0, 3], [0, 2, 0, -1], [0, 0, 1, 5], [0, 0, 0, 1]], np.float32),
                conf=conf, min_consistent=min_consistent)


def edge_cases(seed=0):
    """Known-answer inputs -> list of (name, inputs).  Their fp32 arithmetic is exact or far
    from every threshold, so ``check_fuse(..., exact=True)`` states the kernel's outcome:

    ties          a depth ramp 512 + x/8 + y/16 seen through shifts by odd multiples of 1/64 px:
                  32 xs is a half-integer, the bin follows round-half-even and shows in the
                  reprojected depth 512 + sx/256 + sy/512.  Shifts of -31/64, 31/64 px put
                  coordinates in (-1, 0), (W-1, W) and (H-1, H), where a tap reads 0.
    pixel_tie     constant depth 512, forward shift 3 px and back shift -2 px: dx = 1 exactly,
                  so dx^2 + dy^2 < 1 is False (and 2.5 / -2: dx = 0.5, True).
    saturate      shifts of +-2^30 and +-2^100 px (the bin saturates to int32) and 2^120 px (qx
                  overflows to inf): every tap is off the image, the mask is False.
    qz_zero       a third row of zeros: xs = X / 0 is inf or NaN, the mask is False.
    bad_depths    NaN, 0 and negative depths in the reference and a source; a negative reference
                  depth seen in a negative source is consistent.
    confidence    S = 0, min_consistent = 0: the corner 2x2 blocks, where the upsample is exact,
                  hold proba float32(conf) (rejected) and the next floats above and below.
    """
    rng = np.random.default_rng(seed)
    out = []
    H, W = 12, 16
    yy, xx = np.mgrid[:H, :W].astype(np.float32)
    d512 = np.full((H, W), 512, np.float32)
    ramp = (512 + xx / 8 + yy / 16).astype(np.float32)

    shifts = [(1, 3), (3, -1), (-1, -3), (-3, 5), (-31, 1), (1, -31), (31, 0), (0, 31), (-33, 33)]
    rows = [(shift_rows(a / 64, b / 64), shift_rows(-a / 64, -b / 64)) for a, b in shifts]
    out.append(("ties", _inputs(d512, [ramp] * len(rows), rows, rng)))

    rows = [(shift_rows(3, 0), shift_rows(-2, 0)), (shift_rows(0, 3), shift_rows(0, -2)),
            (shift_rows(2.5, 0), shift_rows(-2, 0)), (shift_rows(-3, 0), shift_rows(2, 0))]
    out.append(("pixel_tie", _inputs(d512, [d512] * len(rows), rows, rng)))

    big = [(2.0 ** 30, 0), (-2.0 ** 30, 0), (0, 2.0 ** 30), (2.0 ** 100, 2.0 ** 100),
           (-2.0 ** 100, 0), (2.0 ** 120, 0)]
    rows = [(shift_rows(a, b), shift_rows(0, 0)) for a, b in big]
    out.append(("saturate", _inputs(d512, [d512] * len(rows), rows, rng)))

    z = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 0]], np.float32).reshape(-1)
    z2 = np.zeros(12, np.float32)
    rows = [(z, shift_rows(0, 0)), (z2, shift_rows(0, 0))]
    out.append(("qz_zero", _inputs(d512, [d512] * 2, rows, rng)))

    dref = d512.copy()
    dref[2, 3], dref[2, 5], dref[3, 7], dref[4, 9] = np.nan, 0, -512, -0.0
    s0 = d512.copy()
    s0[6, 6], s0[6, 10], s0[8, 4] = np.nan, 0, -512
    sneg = -d512
    sh = (shift_rows(0.25, 0.5), shift_rows(-0.25, -0.5))
    out.append(("bad_depths", _inputs(dref, [s0, sneg, d512], [sh, sh, sh], rng)))

    Hc = Wc = 16
    c32 = np.float32(0.999)
    proba = (c32 + rng.uniform(-1e-3, 1e-3, (4, 4))).astype(np.float32)
    proba[0, 0] = c32
    proba[0, 3] = np.nextafter(c32, np.float32(2))
    proba[3, 0] = np.nextafter(c32, np.float32(0))
    proba[3, 3] = c32
    out.append(("confidence", _inputs(np.full((Hc, Wc), 512, np.float32), [], [], rng, proba=proba,
                                      conf=0.999, min_consistent=0)))
    return out


CONF_CORNERS = {(0, 0): False, (0, 1): True, (1, 0): False, (1, 1): False}   # (row, col) of blocks
