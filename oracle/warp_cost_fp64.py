"""Float64 reference of the engine's cost-volume kernels (K1) and their backward, with a
per-element error bound, for per-element checks.

Plain torch only (no casmvsnet_pl_b200 import, no grid_sample): sample positions, bilinear taps
and reductions are written out and evaluated in float64 from the float32 inputs the kernels see
(hypotheses included: a ladder is materialised in float32 with the kernels' two roundings first,
``ops.Ladder.materialize()``).  The same functions run on the CPU and on the GPU; large shapes
are processed in blocks of planes and rows so that peak memory stays near ``BLOCK_BYTES`` plus
two float32 copies of the source features.

Tensors are channels-last: features (B, V, h, w, C), view 0 the reference; projections
(B, V-1, 3, 4); hypotheses (B, D, h, w); cost volumes (B, D, h, w, Cout).

Forward, per reference pixel (x, y), plane d and source view:
    q = R (x, y, 1) + T / d,   u = q_x / q_z,   v = q_y / q_z
q_z <= 1e-7f sends the sample fully outside (behind the camera).  The sample is the bilinear
blend of the zero-padded source image at (u, v) with align_corners semantics (texel centres at
integers), taps nw, ne, sw, se.  Variance: Q/V - (S/V)^2 over the V views (the reference
included); group-wise correlation: the mean over a group of S_c * ref_c over the source views,
divided by V - 1.

Per-element bound |y - y64| <= bound, derived from the kernels' fp32 arithmetic (u = 2^-24):

* Position.  Each of q_x, q_y, q_z is a chain of at most K_Q roundings, each at most u times
  the sum of the absolute terms m = |P0 x| + |P1 y| + |P2| + |P3 / d| (the kernels' chains of
  three fmas have 3; the unfused restatement, three products and three sums, has 6), plus the
  relative error REL_RCP of the reciprocal 1/d (rcp.approx.ftz: 1 ulp = 2^-23; __frcp_rn and
  IEEE division: half of that):  dq <= K_Q u m + REL_RCP |P3 / d|.  Then
      du <= (dq_x + |u| dq_z) / (|q_z| - dq_z) + C_DIV 2^-23 |u|
  where C_DIV covers the reciprocal of q_z (1 ulp) and the product q_x * (1/q_z) (half an ulp);
  dv likewise.
* Sample.  dr <= L (du + dv) + EPS_BLEND sum_i |w_i| |f_i|.  Bilinear interpolation of the
  zero-padded image is Lipschitz with the largest difference of adjacent texels; L is that
  largest difference per channel over the 4x4 texels around the 2x2 window (a position error
  below one texel moves the window by at most one texel), precomputed as a per-texel map by
  max-pooling the difference map and gathered once per sample.  Where du or dv reaches one texel
  the position term is 2 max|f| of the channel instead; where the sample lies outside the image
  by more than du (dv) it is exactly zero for the kernel and the reference alike.  EPS_BLEND
  counts the roundings of the blend: 3 for the weights (1 - f_x, 1 - f_y, their product) and up
  to 7 for the weighted sum (4 products and 3 sums in the unfused form).
* Behind-camera decision.  Where |q_z - 1e-7f| <= dq_z the kernel may keep or drop the sample;
  the bound then allows 2 max|f| of the channel for it, unless every q in the error box
  (q_x +- dq_x, q_y +- dq_y, q_z +- dq_z) projects outside the image: then the sample is exactly
  zero either way.  The same box test, with u' = q_x' / q_z' bounded by the box's corners,
  makes samples next to q_z = 0 (huge u, huge du) exactly zero rather than unbounded.
* Cost.  Variance: sum_v (2/V) |r_v - S/V| dr_v + (1/V) sum_v dr_v^2 (exact to second order;
  the reference view has dr = 0), magnitude A = Q/V + (S/V)^2.  Group-wise correlation:
  sum_{c in g} |ref_c| sum_v dr_{v,c} / (cpg (V-1)), magnitude
  A = sum_{c in g} |ref_c| sum_v m_{v,c} / (cpg (V-1)), m = sum_i |w_i| |f_i| of the sample
  (it bounds every partial sum of S whatever the number of views, and unlike |S| or |r| it does
  not vanish where a sample happens to cross zero).  homo_warp: the sample bound,
  A = sum_i |w_i| |f_i|.  The fp32 reductions add eps A, eps measured per kernel family.  A
  TF32-rounded store adds R_TF32 |y| / (1 - R_TF32) (half an ulp of the unrounded value).
* Gradient of sum(cost * g) with respect to the features, a scatter through the four taps.
  For each contribution coef * w_tap: |coef| (du + dv) onto the 4x4 texels around the window
  (a weight moves by at most du + dv, and the window by at most one texel), and
  (dcoef + eps M) (w_tap + du + dv) onto the taps, M the magnitude of coef (variance:
  |g| (2/V) (|r_v| + sum_u |r_u| / V); group-wise: |coef|), dcoef from the dr above (variance:
  |g| (2/V) (dr_v + sum_u dr_u / V); group-wise: 0).  eps covers the atomic additions in any
  order.  Samples with du or dv >= 1, or an ambiguous behind-camera decision, may land anywhere:
  their |coef| is added to every texel of the view and channel.

Reports (``Report``) give the worst element by err / bound at (b, d, y, x, c) with x % 32, y % 4
(the staged tiles are 32x4, 32x2 or 16x2 pixels) and the plane, the kernel and float64 values,
the bound, the smallest eps that would pass, and the loose share: the fraction of elements whose
bound exceeds LOOSE_REL of their magnitude A, i.e. where the check could not see an error of
that size.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.conv3d_fp64 import R_TF32, TINY, from_blocked, tf32_rna, to_blocked  # noqa: F401

ULP = 2.0 ** -24                    # unit roundoff of fp32
THRESH = float(torch.tensor(1e-7, dtype=torch.float32))   # the kernels' q_z <= 1e-7f
K_Q = 6                             # roundings of one q row (3 fmas; 3 products + 3 sums unfused)
REL_RCP = 2.0 ** -22                # relative error of 1/d: rcp.approx.ftz is within 1 ulp
C_DIV = 2                           # in 2^-23 |u|: rcp.approx of q_z (1) + the product (1/2)
EPS_BLEND = 10 * ULP                # blend: 3 roundings of the weights + 7 of the weighted sum
LOOSE_REL = 0.01                    # loose element: bound > LOOSE_REL * magnitude
BLOCK_BYTES = 1 << 30               # float64 working set per block


# ------------------------------------------------------------------------------- sampling
class _View:
    """One source view of all batch items: zero-padded (2 texels) float32 image, the map of L
    (largest adjacent-texel difference over the 4x4 texels around each window origin), and the
    largest |f| per (b, c)."""

    def __init__(self, f):                                   # f (B, h, w, C) float32
        B, h, w, C = f.shape
        self.h, self.w = h, w
        fp = F.pad(f.float(), (0, 0, 2, 2, 2, 2))            # (B, h+4, w+4, C), exact
        self.f = fp.reshape(B, -1, C)
        fd = fp.double()
        e = torch.zeros_like(fd)
        e[:, :, :-1] = (fd[:, :, 1:] - fd[:, :, :-1]).abs()
        e[:, :-1] = torch.maximum(e[:, :-1], (fd[:, 1:] - fd[:, :-1]).abs())
        # window origin x0 in [-1, w-1] (padded x0+2): its 4x4 neighbourhood is padded x0+1..x0+4
        L = F.max_pool2d(e.permute(0, 3, 1, 2), 4, stride=1)[:, :, :h + 1, :w + 1]
        self.L = (L.permute(0, 2, 3, 1) * (1 + 2.0 ** -22)).float().reshape(B, -1, C)   # round up
        self.fmax = fp.abs().amax(dim=(1, 2)).double()       # (B, C)
        del fd, e


def _positions(P, hyp, y0, h, w):
    """P (B, 3, 4), hyp (B, nd, ny, w) float32 for rows y0.. of an h x w image -> float64
    (B, nd, ny, w) u, v, du, dv, ambiguous, and `zero`: samples that are exactly zero for the
    kernel whatever its rounding (behind the camera, or outside the image for every q within
    the error box: u' = q_x' / q_z' over the box is bounded by its corners)."""
    B = P.shape[0]
    P = P.double().reshape(B, 3, 4, 1, 1, 1)
    inv = 1.0 / hyp.double()
    ny = hyp.shape[2]
    x = torch.arange(w, dtype=torch.float64, device=hyp.device).view(1, 1, 1, w)
    y = torch.arange(y0, y0 + ny, dtype=torch.float64, device=hyp.device).view(1, 1, ny, 1)
    q, dq = [], []
    for i in range(3):
        a, b, c, t = P[:, i, 0] * x, P[:, i, 1] * y, P[:, i, 2], P[:, i, 3] * inv
        q.append(a + b + c + t)
        dq.append(K_Q * ULP * (a.abs() + b.abs() + c.abs() + t.abs()) + REL_RCP * t.abs())
    (qx, qy, qz), (dqx, dqy, dqz) = q, dq
    behind = qz <= THRESH
    amb = (qz - THRESH).abs() <= dqz
    qzs = torch.where(behind, torch.ones_like(qz), qz)
    u = torch.where(behind, torch.full_like(qx, float(w)), qx / qzs)
    v = torch.where(behind, torch.full_like(qy, float(h)), qy / qzs)
    den = (qzs.abs() - dqz).clamp_min(1e-300)
    du = (dqx + u.abs() * dqz) / den + C_DIV * 2.0 ** -23 * u.abs()
    dv = (dqy + v.abs() * dqz) / den + C_DIV * 2.0 ** -23 * v.abs()
    shrink = 1 - C_DIV * 2.0 ** -23
    zlo, zhi = qz - dqz, qz + dqz
    outside = torch.zeros_like(behind)
    for qc, dc, n in ((qx, dqx, w), (qy, dqy, h)):
        lo = torch.minimum((qc - dc) / zlo, (qc - dc) / zhi)
        hi = torch.maximum((qc + dc) / zlo, (qc + dc) / zhi)
        outside |= (zlo > 0) & ((lo * shrink >= n) | (hi * shrink <= -1))
        # q_z' in (1e-7, zhi] or dropped: |q_c'| / q_z' >= (|q_c| - dc) / zhi
        outside |= (zlo <= 0) & ((qc.abs() - dc) * shrink >= (n + 1) * zhi)
    zero = (behind & ~amb) | outside
    return u, v, du, dv, amb, zero


class _Sample:
    """Bilinear samples of one view at flattened positions (B, N): r, dr, m = sum |w||f|
    (B, N, C) float64, plus what the backward scatters: tap base index, weights, near/far."""

    def __init__(self, view, u, v, du, dv, amb, zero, grad=False):
        h, w = view.h, view.w
        B = u.shape[0]
        u, v, du, dv, amb, zero = (t.reshape(B, -1) for t in (u, v, du, dv, amb, zero))
        bi = torch.arange(B, device=u.device).view(B, 1)
        xf, yf = torch.floor(u), torch.floor(v)
        fx, fy = u - xf, v - yf
        inside = ~(zero & ~amb) & (u > -1) & (u < w) & (v > -1) & (v < h)
        x0 = xf.clamp(-2, w).long()
        y0 = yf.clamp(-2, h).long()
        base = (y0 + 2) * (w + 4) + (x0 + 2)
        wts = [(1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy]
        wts = [torch.where(inside, t, torch.zeros_like(t)) for t in wts]
        offs = [0, 1, w + 4, w + 5]                          # nw, ne, sw, se
        # texel scale for the loose share: the window anchored inside the image, so that a
        # sample exactly on the border (u = w, weight 0 on every texel) still has one
        xc, yc = x0.clamp(-1, w - 1), y0.clamp(-1, h - 1)
        tbase = (yc + 2) * (w + 4) + (xc + 2)
        r = m = tx = 0
        for wt, o in zip(wts, offs):
            t = view.f[bi, base + o].double()
            r = r + wt.unsqueeze(-1) * t
            m = m + wt.unsqueeze(-1) * t.abs()
            tx = tx + view.f[bi, tbase + o].double().abs()
        lo = (yc + 1) * (w + 1) + (xc + 1)
        L = view.L[bi, lo].double()
        duv = (du + dv).unsqueeze(-1)
        pe = L * duv
        far = ((du >= 1) | (dv >= 1)).unsqueeze(-1)
        fm = view.fmax.unsqueeze(1)
        pe = torch.where(far, 2 * fm, pe)
        zero = (zero | (((u + du <= -1) | (u - du >= w) | (v + dv <= -1) | (v - dv >= h)) & ~amb))
        zero = zero.unsqueeze(-1)
        pe = torch.where(zero, torch.zeros_like(pe), pe)
        pe = torch.where(amb.unsqueeze(-1), 2 * fm, pe)
        self.r, self.m, self.t = r, m, tx
        self.dr = pe + EPS_BLEND * m
        if grad:
            self.base, self.wts, self.duv = base, wts, duv
            self.nb = (yc + 1) * (w + 4) + (xc + 1)
            self.live = ~zero
            self.near = ~zero.squeeze(-1) & ~far.squeeze(-1) & ~amb
            self.anywhere = (far.squeeze(-1) | amb) & ~zero.squeeze(-1)


def _blocks(B, D, h, w, per_px):
    """(d0, d1, y0, y1) blocks of at most BLOCK_BYTES, per_px float64 per (b, plane, pixel)."""
    px = max(1, BLOCK_BYTES // (8 * per_px * B))
    if px >= h * w:
        nd = max(1, min(D, px // (h * w)))
        for d0 in range(0, D, nd):
            yield d0, min(D, d0 + nd), 0, h
    else:
        ny = max(1, px // w)
        for d0 in range(D):
            for y0 in range(0, h, ny):
                yield d0, d0 + 1, y0, min(h, y0 + ny)


# ------------------------------------------------------------------------------- reports
class Report:
    """Worst element and loose share of one check, accumulated over blocks."""

    def __init__(self, eps, tf32, names):
        self.eps, self.tf32, self.names = eps, tf32, names
        self.ratio = -1.0
        self.eps_needed = 0.0
        self.loose = 0
        self.n = 0
        self.worst = None

    def add(self, y, y64, bound0, A, origin, scale):
        y = y.to(device=y64.device, dtype=torch.float64)
        err = (y - y64).abs()
        slack = bound0 + TINY
        if self.tf32:
            slack = slack + R_TF32 * y.abs() / (1 - R_TF32)
        bound = slack + self.eps * A
        nan = torch.isnan(y)
        ratio = torch.where(nan, torch.full_like(err, float("inf")), err / bound)
        over = (err - slack).clamp_min(0)
        need = torch.where(over > 0, over / A, torch.zeros_like(over))
        need = torch.where(nan, torch.full_like(need, float("inf")), need)
        self.eps_needed = max(self.eps_needed, float(need.max()))
        self.loose += int((bound0 + self.eps * A > LOOSE_REL * scale).sum())
        self.n += y.numel()
        flat = int(torch.argmax(ratio.reshape(-1)))
        rmax = float(ratio.reshape(-1)[flat])
        if rmax > self.ratio or self.worst is None:
            idx = []
            for n in reversed(y.shape):
                idx.append(flat % n)
                flat //= n
            idx = list(reversed(idx))
            at = tuple(int(i + o) for i, o in zip(idx, origin))
            i = tuple(idx)
            self.ratio = rmax
            self.worst = dict(at=at, got=float(y[i]), want=float(y64[i]), bound=float(bound[i]),
                              A=float(A[i]))

    @property
    def ok(self):
        return self.eps_needed <= self.eps

    @property
    def loose_share(self):
        return self.loose / max(1, self.n)

    def describe(self):
        wv = self.worst
        at = dict(zip(self.names, wv["at"]))
        where = ", ".join(f"{k}={v}" for k, v in at.items())
        extra = ""
        if "x" in at and "y" in at:
            extra = f" x%32={at['x'] % 32} y%4={at['y'] % 4}"
        if "d" in at:
            extra += f" plane={at['d']}"
        return (f"worst err/bound {self.ratio:.3e} at ({where}){extra}: got {wv['got']!r}, "
                f"float64 {wv['want']!r}, bound {wv['bound']:.3e}, A {wv['A']:.3e}; "
                f"eps needed {self.eps_needed:.3e} (eps {self.eps:.3e}); "
                f"loose share {self.loose_share:.2e}")


# ------------------------------------------------------------------------------- forward
def _cost_blocks(feats, proj, hyp, num_groups, mode):
    """Yields (d0, y0, y64, bound0, A) per block, (B, nd, ny, w, Cout) float64.  mode: "var",
    "gwc" or "homo" (feats (B, 1 + 1, ...) then: view 1 is warped, view 0 ignored)."""
    B, V, h, w, C = feats.shape
    D = hyp.shape[1]
    views = [_View(feats[:, v]) for v in range(1, V)]
    ref_all = feats[:, 0].double() if mode != "homo" else None
    per_px = C * (2 * V + 10)
    for d0, d1, y0, y1 in _blocks(B, D, h, w, per_px):
        nd, ny = d1 - d0, y1 - y0
        hb = hyp[:, d0:d1, y0:y1].contiguous()
        samples = []
        for v in range(V - 1):
            pos = _positions(proj[:, v], hb, y0, h, w)
            samples.append(_Sample(views[v], *pos))
            del pos
        shape = (B, nd, ny, w)
        if mode == "homo":
            s = samples[0]
            y64, bound0, A, scale = s.r, s.dr, s.m, s.t
            cout = C
        else:
            ref = ref_all[:, y0:y1].reshape(B, 1, ny * w, C).expand(B, nd, ny * w, C)
            ref = ref.reshape(B, -1, C)
            if mode == "var":
                S = ref + sum(s.r for s in samples)
                Q = ref * ref + sum(s.r * s.r for s in samples)
                mean = S / V
                y64 = Q / V - mean * mean
                bound0 = sum((2.0 / V) * (s.r - mean).abs() * s.dr + s.dr * s.dr / V
                             for s in samples)
                A = Q / V + mean * mean
                scale = (ref * ref + sum(s.t * s.t for s in samples)) / V
                cout = C
            else:
                G = num_groups
                cpg = C // G
                k = 1.0 / (cpg * (V - 1))
                S = sum(s.r for s in samples)
                aref = ref.abs()
                y64 = (S * ref).reshape(B, -1, G, cpg).sum(-1) * k
                bound0 = (aref * sum(s.dr for s in samples)).reshape(B, -1, G, cpg).sum(-1) * k
                A = (aref * sum(s.m for s in samples)).reshape(B, -1, G, cpg).sum(-1) * k
                scale = (aref * sum(s.t for s in samples)).reshape(B, -1, G, cpg).sum(-1) * k
                cout = G
        yield d0, y0, *(t.reshape(*shape, cout) for t in (y64, bound0, A, scale))
        del samples


def cost_ref(feats, proj, hyp, num_groups=1):
    """Float64 cost volume (B, D, h, w, Cout) and its bound without eps (bound0) and magnitude
    A, whole (small shapes)."""
    return _whole(_cost_blocks(feats, proj, hyp, num_groups, "var" if num_groups == 1 else "gwc"),
                  hyp.shape)[:3]


def homo_warp_ref(src, proj, hyp):
    """src (B, h, w, C), proj (B, 3, 4) -> float64 warped (B, D, h, w, C), bound0, A."""
    f = torch.stack([src, src], 1)
    return _whole(_cost_blocks(f, proj.unsqueeze(1), hyp, 1, "homo"), hyp.shape)[:3]


def _whole(gen, hshape):
    B, D, h, w = hshape
    out = None
    for d0, y0, *ts in gen:
        if out is None:
            out = [t.new_zeros(B, D, h, w, t.shape[-1]) for t in ts]
        for o, t in zip(out, ts):
            o[:, d0:d0 + t.shape[1], y0:y0 + t.shape[2]] = t
    return tuple(out)


@torch.no_grad()
def check_cost(y, feats, proj, hyp, num_groups, eps, tf32=False):
    """Kernel cost volume y (B, D, h, w, Cout), channels-last, against float64."""
    rep = Report(eps, tf32, ("b", "d", "y", "x", "c"))
    mode = "var" if num_groups == 1 else "gwc"
    for d0, y0, y64, b0, A, scale in _cost_blocks(feats, proj, hyp, num_groups, mode):
        yb = y[:, d0:d0 + y64.shape[1], y0:y0 + y64.shape[2]]
        rep.add(yb, y64, b0, A, (0, d0, y0, 0, 0), scale)
    return rep


@torch.no_grad()
def check_homo_warp(y, src, proj, hyp, eps):
    """Kernel homo_warp output y (B, D, h, w, C) against float64."""
    rep = Report(eps, False, ("b", "d", "y", "x", "c"))
    f = torch.stack([src, src], 1)
    for d0, y0, y64, b0, A, scale in _cost_blocks(f, proj.unsqueeze(1), hyp, 1, "homo"):
        rep.add(y[:, d0:d0 + y64.shape[1], y0:y0 + y64.shape[2]], y64, b0, A, (0, d0, y0, 0, 0),
                scale)
    return rep


# ------------------------------------------------------------------------------- backward
@torch.no_grad()
def warp_cost_bwd_ref(feats, proj, hyp, gcost, num_groups):
    """Gradient of sum(cost * gcost) with respect to feats (B, V, h, w, C), float64, with its
    bound without eps (bound0) and the magnitude M of the eps term, all (B, V, h, w, C)."""
    B, V, h, w, C = feats.shape
    D = hyp.shape[1]
    G = num_groups
    gwc = G > 1
    cpg = C // G if gwc else 1
    k = 1.0 / (cpg * (V - 1)) if gwc else 0.0
    dev = feats.device
    npad = (h + 4) * (w + 4)
    views = [_View(feats[:, v]) for v in range(1, V)]
    acc = {n: torch.zeros(B * npad * (V - 1), C, dtype=torch.float64, device=dev)
           for n in ("g", "b", "m", "s")}
    anywhere = torch.zeros(B, V - 1, C, dtype=torch.float64, device=dev)
    gref = torch.zeros(B, h * w, C, dtype=torch.float64, device=dev)
    bref = torch.zeros_like(gref)
    mref = torch.zeros_like(gref)
    sref = torch.zeros_like(gref)
    ref_all = feats[:, 0].double().reshape(B, h * w, C)
    offs = [0, 1, w + 4, w + 5]
    for d0, d1, y0, y1 in _blocks(B, D, h, w, C * (2 * V + 16)):
        nd, ny = d1 - d0, y1 - y0
        hb = hyp[:, d0:d1, y0:y1].contiguous()
        ss = [_Sample(views[v], *_positions(proj[:, v], hb, y0, h, w), grad=True) for v in range(V - 1)]
        ref = ref_all[:, y0 * w:y1 * w].reshape(B, 1, ny * w, C).expand(B, nd, ny * w, C)
        ref = ref.reshape(B, -1, C)
        g = gcost[:, d0:d1, y0:y1].double().reshape(B, -1, gcost.shape[-1])
        if gwc:
            g = g.repeat_interleave(cpg, dim=-1)
            S = sum(s.r for s in ss)
            gr, br = g * S * k, g.abs() * sum(s.dr for s in ss) * k
            mr = g.abs() * sum(s.m for s in ss) * k
            sr = g.abs() * sum(s.t for s in ss) * k
        else:
            mean = (ref + sum(s.r for s in ss)) / V
            sdr = sum(s.dr for s in ss) / V
            sabs = (ref.abs() + sum(s.r.abs() for s in ss)) / V
            gr = g * (2.0 / V) * (ref - mean)
            br = g.abs() * (2.0 / V) * sdr
            mr = g.abs() * (2.0 / V) * (ref.abs() + sabs)
            sr = g.abs() * (2.0 / V) * (ref.abs() + (ref.abs() + sum(s.t for s in ss)) / V)
        for t, a in ((gr, gref), (br, bref), (mr, mref), (sr, sref)):
            a[:, y0 * w:y1 * w] += t.reshape(B, nd, ny * w, C).sum(1)
        for v, s in enumerate(ss):
            if gwc:
                coef = g * ref * k
                dcoef = torch.zeros_like(coef)
                mc = coef.abs()
            else:
                coef = g * (2.0 / V) * (s.r - mean)
                dcoef = g.abs() * (2.0 / V) * (s.dr + sdr)
                mc = g.abs() * (2.0 / V) * (s.r.abs() + sabs)
            bofs = (torch.arange(B, device=dev).view(B, 1) * (V - 1) + v) * npad
            for wt, o in zip(s.wts, offs):
                idx = (bofs + s.base + o).reshape(-1)
                wt = wt.unsqueeze(-1)
                spread = torch.where(s.live, wt + s.duv, torch.zeros_like(s.duv))
                acc["g"].index_add_(0, idx, (coef * wt).reshape(-1, C))
                acc["b"].index_add_(0, idx, (dcoef * spread).reshape(-1, C))
                acc["m"].index_add_(0, idx, (mc * spread).reshape(-1, C))
            pos = torch.where(s.near.unsqueeze(-1), coef.abs() * s.duv, torch.zeros_like(coef))
            pos = pos.reshape(-1, C)
            reach = torch.where(s.near.unsqueeze(-1), mc, torch.zeros_like(mc)).reshape(-1, C)
            for dy in range(4):
                for dx in range(4):
                    idx = (bofs + s.nb + dy * (w + 4) + dx).reshape(-1)
                    acc["b"].index_add_(0, idx, pos)
                    acc["s"].index_add_(0, idx, reach)
            far = s.anywhere.unsqueeze(-1)
            anywhere[:, v] += torch.where(far, coef.abs() + dcoef, torch.zeros_like(coef)).sum(1)
        del ss
    out = []
    for n, r in (("g", gref), ("b", bref), ("m", mref), ("s", sref)):
        src = acc[n].reshape(B, V - 1, h + 4, w + 4, C)[:, :, 2:h + 2, 2:w + 2]
        if n == "b":
            src = src + anywhere.view(B, V - 1, 1, 1, C)
        out.append(torch.cat([r.reshape(B, 1, h, w, C), src], 1))
    return tuple(out)


@torch.no_grad()
def check_warp_cost_bwd(gf, feats, proj, hyp, gcost, num_groups, eps):
    """Kernel feature gradient gf (B, V, h, w, C) against float64."""
    g64, b0, M, scale = warp_cost_bwd_ref(feats, proj, hyp, gcost, num_groups)
    rep = Report(eps, False, ("b", "view", "y", "x", "c"))
    rep.add(gf, g64, b0, M, (0, 0, 0, 0, 0), scale)
    return rep
