"""Float64 reference of the Poisson kernels (csrc/poisson.cu) with a per-element admissible error,
for per-element checks at every depth and multigrid level.

oracle/poisson_oracle.py restates the kernels' float32 rule; this module does not.  Each check
takes one kernel call's own inputs and outputs, applies the operation in float64 (torch, on the
inputs' device) and returns a Report: ``ok``, ``eps_needed`` (the worst |got - ref| / unit over the
checked elements, where the admissible error is ``eps * unit``) and the worst location, as
(level, x, y, z) for grid fields and (point,) or (cell,) otherwise.  u = 2^-24.

Grid fields are given as (n, n, n) or (n, n, n, 3) views, numpy or torch, on any device.  Every
stage is local (stencil radius <= 2), so each check takes a list of windows, boxes
(x0, y0, z0, x1, y1, z1) of nodes of the checked level, and reads only the window and a halo:
depths 9 and 10 are checked without a host copy of a field.  ``windows(n, ...)`` builds the list
the tests use: the eight corners (the upper Dirichlet face and coarse index n - 1), the face
centres, given surface nodes, and the last x-slabs (at depth 10 a V offset past 2^31 floats).

Rules and bounds, per kernel:

* Levels.  Level l has n = N >> l nodes per axis.  The finest level's interior is 1..n-2; a
  coarse level's interior is 1..n-1 and its index n, which is not stored, reads as 0.  Outside the
  interior a smoothed or prolonged field is unchanged and a residual or restriction is 0 exactly.
* smooth (one red-black sweep).  Red nodes (x + y + z even) take (nbsum(e) - h^2 r) / 6 of the
  call's input e; black nodes take it of the input with the red nodes replaced by the call's own
  red output.  unit = (sum |neighbours| + h^2 |r|) / 6, eps 8u (5 adds, h*h, h2 r, the
  subtraction and the division).
* mg_residual.  r - (nbsum(e) - 6 e) / h^2; unit = |r| + (sum |nb| + 6 |e|) / h^2, eps 10u.
* restrict.  Coarse interior I = sum over fine 2I + {-1,0,1}^3 of (1/4, 1/2, 1/4)^3 weights;
  products are exact, 26 adds: unit = sum w |f|, eps 27u.
* prolong_add.  Fine interior p += trilinear coarse value, coarse I at fine 2I, index nc reads 0;
  unit = |f| + sum w |c|, eps 9u.
* accumulate.  chi + e in double: unit = |chi| + |e|, eps 2^-52.
* rhs, residual.  One double stencil rounded once to float32: unit = |ref| + 2^-25 T, where T is
  the sum of the stencil's |terms|, eps u (the double error, below 16 2^-53 T, fits 2^-49 T).
* Reductions (||b||^2, ||r||^2, the iso sum).  |got - fsum(terms)| <= n 2^-52 sum |terms| (plus
  the terms' own allowance where they are double intermediates the kernel does not store).
  fsum is math.fsum up to 2^22 terms and a float64 torch sum, with its pairwise bound, above.
* cell_keys.  q = p / h in double.  Where float32(q) == q (the kernel's division is exact) the
  cell is rint(q), half to even.  Otherwise the admissible cells are rint(q -+ ulp32(q)): one
  cell, or both sides within one float32 ulp of a tie.  A key is none where a coordinate is not
  finite, the normal has length 0 or is not finite, or the cell may lie outside 0..N-1.  Unit
  normals: float32(x / |n|), unit |x / |n|| + 2^-26, eps u; 0 where not usable.
* splat, iso.  The weight of node k is the hat product prod_a max(0, 1 - |q_a - k_a|), which is
  the trilinear weight of either floor corner set and continuous in q.  |q32 - q64| <= u |q| and
  frac adds at most 2u, so per axis the hat lies within delta = u (|q| + 2) (1 + 2^-20); the
  float32 weight lies in [prod lo (1 - 3u), prod hi (1 + 3u)] of the clipped per-axis intervals,
  to first order |w - w64| <= 3u (1 + |q| |dw/dq|).  V, W, C are float32 roundings of sums of
  admissible weights times the point's normal or colour: err <= e + u (|X64| + e) + 2^-48 A,
  unit = that / u, eps u.  The iso value uses the same weights against the kernel's chi.
* cell_moments.  Double sums of d = p - centre: unit = count * sum |terms|, eps 2^-51.
* cell_normals.  The block of 3x3x3 cells summed, covariance m/m0 - mu mu^T, np.linalg.eigh.
  With S the raw second moment's trace / m0 and gap = l1 - l0, the normal must lie within
  angle K 2^-52 S / gap of the l0 eigenvector (K = 64): eps_needed = sin(angle) gap / S, eps
  K 2^-52.  Cells with gap <= GAP_FLOOR S are exempt and counted.  The rank decision
  (l2 > 0 and l1 > 1e-10 l2) is admissible on either side within K 2^-52 S of its threshold.
  Blocks of fewer than 3 points are dropped with normal 0.
* orient.  The nearest camera by the kernel's own double distance (each operation rounded, so
  the values are reproducible exactly); an exact tie goes to the lower index, a near tie within
  4 2^-52 d2 to either.  The output is float32(+-cn) with sign of n . (C - p), either sign where
  |dot| <= 4 2^-52 sum |n_a (C_a - p_a)|.
* trim, brick_flags.  keep = any W > 0 within the 5x5x5 box, flags = any kept node per 8^3 brick
  of global nodes: exact.
* fill_bricks, fill_tsdf.  Weight 1 at kept in-grid voxels and 0 elsewhere, exact; colour
  box5(C) / box5(W) (W, C >= 0, so the double sums do not cancel): unit |ref|, eps u (1 + 2^-20);
  tsdf = float32(chi - iso): unit |ref| + 2^-28 (|chi| + |iso|), eps u.
"""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
SAFE = 1 + 2.0 ** -20
RANK_EPS = 1e-10
K_EIG = 64
GAP_FLOOR = 1e-8
KEY_NONE = np.iinfo(np.int64).max
COARSEST = 8
EPS = dict(smooth=8 * U, mg_residual=10 * U, restrict=27 * U, prolong_add=9 * U,
           accumulate=2.0 ** -52, residual=U * SAFE, rhs=U * SAFE, reduction=2.0 ** -52,
           cell_keys=U * SAFE, splat=U, iso=U, iso_sum=2.0 ** -52, moments=2.0 ** -51,
           normals=K_EIG * 2.0 ** -52, orient=0.0, trim=0.0, brick_flags=0.0,
           fill_bricks=U * SAFE, fill_tsdf=U * SAFE)


# ------------------------------------------------------------------------------- reports
class Report:
    """Worst eps needed of one kernel over the checked elements and windows, where it was, and
    how many elements failed, were checked and were exempt."""

    def __init__(self, kernel, eps=None):
        self.kernel = kernel
        self.eps = EPS[kernel] if eps is None else eps
        self.eps_needed = 0.0
        self.where = None
        self.bad = 0
        self.checked = 0
        self.exempt = 0
        self.first_bad = None

    def add(self, need, origin=(), prefix=()):
        """need: per-element eps needed (any shape, its index + origin is the location)."""
        need = torch.nan_to_num(torch.as_tensor(need).double(), nan=float("inf"))
        if need.numel() == 0:
            return
        self.checked += need.numel()
        bad = need > self.eps
        nb = int(bad.sum())
        if nb and self.first_bad is None:
            self.first_bad = self._loc(bad.nonzero()[0], origin, prefix)
        self.bad += nb
        m = float(need.max())
        if m > self.eps_needed or self.where is None:
            idx = np.unravel_index(int(torch.argmax(need.reshape(-1))), tuple(need.shape))
            self.eps_needed = max(self.eps_needed, m)
            self.where = self._loc(idx, origin, prefix)

    def mismatch(self, bad, origin=(), prefix=()):
        """Discrete outcomes: bad marks elements outside their admissible set."""
        bad = torch.as_tensor(bad).bool()
        self.add(torch.where(bad, float("inf"), 0.0).double(), origin, prefix)

    @staticmethod
    def _loc(idx, origin, prefix):
        idx = [int(v) for v in idx]
        o = list(origin) + [0] * (len(idx) - len(origin))
        return tuple(prefix) + tuple(a + b for a, b in zip(idx, o))[:max(len(origin), 1)]

    @property
    def ok(self):
        return self.bad == 0

    def merge(self, other):
        if other.eps_needed > self.eps_needed or self.where is None:
            self.eps_needed, self.where = other.eps_needed, other.where
        if other.bad and self.first_bad is None:
            self.first_bad = other.first_bad
        self.bad += other.bad
        self.checked += other.checked
        self.exempt += other.exempt
        return self

    def describe(self):
        return (f"{self.kernel}: eps needed {self.eps_needed:.3e} (eps {self.eps:.3e}) at "
                f"{self.where}; {self.bad} bad of {self.checked}"
                + (f", first at {self.first_bad}" if self.bad else "")
                + (f", {self.exempt} exempt" if self.exempt else ""))


# ------------------------------------------------------------------------------- windows
def full(n):
    return (0, 0, 0, n, n, n)


def windows(n, size=32, surface=(), slabs=True):
    """Boxes of nodes of a level of n per axis: the eight corners, the six face centres, a box
    around each of the `surface` nodes and (``slabs``) the last two x-slabs of size x n x size
    strips at their y, z corners and centre.  All clipped to the grid; a grid no larger than the
    box is one window."""
    s = min(size, n)
    if s == n:
        return [full(n)]
    out = []
    for cx in (0, n - s):
        for cy in (0, n - s):
            for cz in (0, n - s):
                out.append((cx, cy, cz, cx + s, cy + s, cz + s))
    m = (n - s) // 2
    for a in range(3):
        for side in (0, n - s):
            c = [m, m, m]
            c[a] = side
            out.append((c[0], c[1], c[2], c[0] + s, c[1] + s, c[2] + s))
    for p in surface:
        c = [min(max(int(v) - s // 2, 0), n - s) for v in p]
        out.append((c[0], c[1], c[2], c[0] + s, c[1] + s, c[2] + s))
    if slabs:
        x0 = max(n - 2, 0)
        out.append((x0, 0, 0, n, n, min(8, n)))
        out.append((x0, 0, n - min(8, n), n, n, n))
    return out


def _t(a, dev=None):
    t = a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
    return t if dev is None else t.to(dev)


def fetch(a, lo, hi, dev=None):
    """Box [lo, hi) of a (n, n, n[, c]) field as float64 on dev (default: a's device); entries
    outside 0..n-1 read 0."""
    a = _t(a)
    n = a.shape[0]
    dev = a.device if dev is None else dev
    shape = tuple(h - l for l, h in zip(lo, hi)) + tuple(a.shape[3:])
    out = torch.zeros(shape, dtype=torch.float64, device=dev)
    c0 = [max(l, 0) for l in lo]
    c1 = [min(h, n) for h in hi]
    if all(b > a_ for a_, b in zip(c0, c1)):
        src = a[c0[0]:c1[0], c0[1]:c1[1], c0[2]:c1[2]]
        out[c0[0] - lo[0]:c1[0] - lo[0], c0[1] - lo[1]:c1[1] - lo[1],
            c0[2] - lo[2]:c1[2] - lo[2]] = src.to(dev).double()
    return out


def _grid_xyz(w, dev):
    ax = [torch.arange(w[a], w[a + 3], device=dev) for a in range(3)]
    return torch.meshgrid(*ax, indexing="ij")


def interior(w, n, level, dev):
    """Mask of the window's nodes in the level's interior."""
    top = n if level else n - 1
    x, y, z = _grid_xyz(w, dev)
    return (x > 0) & (y > 0) & (z > 0) & (x < top) & (y < top) & (z < top)


def _nbs(P):
    """Neighbour sum and sum of |neighbours| of the inner nodes of a box padded by 1."""
    i = slice(1, -1)
    terms = (P[:-2, i, i], P[2:, i, i], P[i, :-2, i], P[i, 2:, i], P[i, i, :-2], P[i, i, 2:])
    return sum(terms), sum(t.abs() for t in terms)


def _need(got, ref, unit):
    err = (got - ref).abs()
    q = err / unit
    return torch.where(err == 0, torch.zeros_like(q), q)


def _same(got, ref):
    """Exact equality outside the stencil's support (NaN never equal)."""
    return ~(got == ref)


def _pad(w, r):
    return (w[0] - r, w[1] - r, w[2] - r), (w[3] + r, w[4] + r, w[5] + r)


# ------------------------------------------------------------------------------- multigrid kernels
def check_smooth(e0, e1, r, n, level, h, wins=None, rep=None, zero_first=False):
    """One red-black sweep (sweeps = 1) of poisson_smooth: e0 the field before (ignored with
    zero_first, which starts from 0), e1 after."""
    rep = rep or Report("smooth")
    h = float(np.float32(h))
    for w in wins or [full(n)]:
        dev = _t(e1).device
        lo, hi = _pad(w, 1)
        E1 = fetch(e1, lo, hi)
        E0 = torch.zeros_like(E1) if zero_first else fetch(e0, lo, hi, dev)
        R = fetch(r, w[:3], w[3:], dev)
        x, y, z = [torch.arange(lo[a], hi[a], device=dev) for a in range(3)]
        red = ((x[:, None, None] + y[None, :, None] + z[None, None, :]) % 2) == 0
        E = torch.where(red, E1, E0)                  # red from the call, black from its input
        s, sa = _nbs(E)
        ref = (s - h * h * R) / 6
        unit = (sa + h * h * R.abs()) / 6
        inner = interior(w, n, level, dev)
        got = E1[1:-1, 1:-1, 1:-1]
        need = torch.where(inner, _need(got, ref, unit), 0.0)
        need = torch.where(~inner & _same(got, E0[1:-1, 1:-1, 1:-1]), float("inf"), need)
        rep.add(need, w[:3], (level,))
    return rep


def check_mg_residual(e, r, out, n, level, h, wins=None, rep=None):
    rep = rep or Report("mg_residual")
    h = float(np.float32(h))
    for w in wins or [full(n)]:
        dev = _t(out).device
        lo, hi = _pad(w, 1)
        E = fetch(e, lo, hi, dev)
        R = fetch(r, w[:3], w[3:], dev)
        s, sa = _nbs(E)
        c = E[1:-1, 1:-1, 1:-1]
        ref = R - (s - 6 * c) / (h * h)
        unit = R.abs() + (sa + 6 * c.abs()) / (h * h)
        inner = interior(w, n, level, dev)
        got = fetch(out, w[:3], w[3:], dev)
        need = torch.where(inner, _need(got, ref, unit), 0.0)
        need = torch.where(~inner & (got != 0), float("inf"), need)
        rep.add(need, w[:3], (level,))
    return rep


def _apply3(Ms, A):
    """Apply one matrix per axis to a 3-D box (separably)."""
    A = torch.einsum("ia,abc->ibc", Ms[0], A)
    A = torch.einsum("jb,ibc->ijc", Ms[1], A)
    return torch.einsum("kc,ijc->ijk", Ms[2], A)


def _restrict_matrix(c0, c1, f0, f1, nc, dev, weights=(0.25, 0.5, 0.25)):
    """(c1 - c0, f1 - f0) full-weighting rows of coarse interior nodes c0..c1-1."""
    M = torch.zeros(c1 - c0, f1 - f0, dtype=torch.float64, device=dev)
    for i, I in enumerate(range(c0, c1)):
        if 1 <= I <= nc - 1:
            for d, wt in zip((-1, 0, 1), weights):
                M[i, 2 * I + d - f0] = wt
    return M


def check_restrict(f, c, nf, level_c=1, wins=None, rep=None):
    """poisson_restrict: fine f (nf^3) -> coarse c (nc^3); wins are coarse boxes."""
    rep = rep or Report("restrict")
    nc = nf // 2
    for w in wins or [full(nc)]:
        dev = _t(c).device
        flo = [2 * v - 1 for v in w[:3]]
        fhi = [2 * v for v in w[3:]]
        F = fetch(f, flo, fhi, dev)
        Ms = [_restrict_matrix(w[a], w[a + 3], flo[a], fhi[a], nc, dev) for a in range(3)]
        ref = _apply3(Ms, F)
        unit = _apply3(Ms, F.abs())
        got = fetch(c, w[:3], w[3:], dev)
        inner = interior(w, nc, 1, dev)
        need = torch.where(inner, _need(got, ref, unit), 0.0)
        need = torch.where(~inner & (got != 0), float("inf"), need)
        rep.add(need, w[:3], (level_c,))
    return rep


def _prolong_matrix(p0, p1, c0, c1, dev):
    M = torch.zeros(p1 - p0, c1 - c0, dtype=torch.float64, device=dev)
    for i, p in enumerate(range(p0, p1)):
        if p % 2 == 0:
            M[i, p // 2 - c0] = 1.0
        else:
            M[i, p // 2 - c0] = 0.5
            M[i, p // 2 + 1 - c0] = 0.5
    return M


def check_prolong_add(c, f0, f1, nc, fine_level, wins=None, rep=None):
    """poisson_prolong_add: f1 = f0 + prolong(c) at the fine level's interior; wins are fine."""
    rep = rep or Report("prolong_add")
    nf = 2 * nc
    for w in wins or [full(nf)]:
        dev = _t(f1).device
        clo = [v // 2 for v in w[:3]]
        chi_ = [(v - 1) // 2 + 2 for v in w[3:]]
        C = fetch(c, clo, chi_, dev)
        Ms = [_prolong_matrix(w[a], w[a + 3], clo[a], chi_[a], dev) for a in range(3)]
        add = _apply3(Ms, C)
        mag = _apply3(Ms, C.abs())
        F0 = fetch(f0, w[:3], w[3:], dev)
        got = fetch(f1, w[:3], w[3:], dev)
        inner = interior(w, nf, fine_level, dev)
        need = torch.where(inner, _need(got, F0 + add, F0.abs() + mag), 0.0)
        need = torch.where(~inner & _same(got, F0), float("inf"), need)
        rep.add(need, w[:3], (fine_level,))
    return rep


def check_accumulate(chi0, e, chi1, n, wins=None, rep=None):
    rep = rep or Report("accumulate")
    for w in wins or [full(n)]:
        dev = _t(chi1).device
        a, b = fetch(chi0, w[:3], w[3:], dev), fetch(e, w[:3], w[3:], dev)
        got = fetch(chi1, w[:3], w[3:], dev)
        rep.add(_need(got, a + b, a.abs() + b.abs()), w[:3], (0,))
    return rep


def _stencil_need(got, ref, T):
    return _need(got, ref, ref.abs() + 2.0 ** -25 * T)


def check_residual(chi, b, r, N, h, wins=None, rep=None):
    """poisson_residual: r = float32(b - (nbsum(chi) - 6 chi) / h^2) at the interior, double chi.
    -> report, and per window the float64 residual (for the ||r||^2 check)."""
    rep = rep or Report("residual")
    h = float(np.float32(h))
    parts = []
    for w in wins or [full(N)]:
        dev = _t(r).device
        lo, hi = _pad(w, 1)
        X = fetch(chi, lo, hi, dev)
        B = fetch(b, w[:3], w[3:], dev)
        s, sa = _nbs(X)
        c = X[1:-1, 1:-1, 1:-1]
        inner = interior(w, N, 0, dev)
        ref = torch.where(inner, B - (s - 6 * c) / (h * h), 0.0)
        T = torch.where(inner, B.abs() + (sa + 6 * c.abs()) / (h * h), 0.0)
        got = fetch(r, w[:3], w[3:], dev)
        need = torch.where(inner, _stencil_need(got, ref, T), 0.0)
        need = torch.where(~inner & (got != 0), float("inf"), need)
        rep.add(need, w[:3], (0,))
        parts.append((ref, T))
    return rep, parts


def check_rhs(V, b, N, h, wins=None, rep=None):
    """poisson_rhs: b = float32(div V / (2h)) at the interior, 0 on the outer layer."""
    rep = rep or Report("rhs")
    h = float(np.float32(h))
    for w in wins or [full(N)]:
        dev = _t(b).device
        lo, hi = _pad(w, 1)
        P = fetch(V, lo, hi, dev)
        i = slice(1, -1)
        terms = (P[2:, i, i, 0], -P[:-2, i, i, 0], P[i, 2:, i, 1], -P[i, :-2, i, 1],
                 P[i, i, 2:, 2], -P[i, i, :-2, 2])
        d = ((terms[0] + terms[1]) + (terms[2] + terms[3])) + (terms[4] + terms[5])
        T = sum(t.abs() for t in terms) / (2 * h)
        ref = d / (2 * h)
        inner = interior(w, N, 0, dev)
        got = fetch(b, w[:3], w[3:], dev)
        need = torch.where(inner, _stencil_need(got, ref, T), 0.0)
        need = torch.where(~inner & (got != 0), float("inf"), need)
        rep.add(need, w[:3], (0,))
    return rep


def fsum(t):
    """(exact-ish sum of t, its own error bound): math.fsum up to 2^22 terms, else a float64
    torch sum with the pairwise bound (log2 n + 1) 2^-53 sum |t|."""
    t = _t(t).double().reshape(-1)
    if t.numel() <= 1 << 22:
        return math.fsum(t.cpu().numpy().tolist()), 0.0
    return float(t.sum()), (math.log2(t.numel()) + 1) * 2.0 ** -53 * float(t.abs().sum())


def check_reduction(got, terms, extra=0.0, rep=None, name="reduction"):
    """A kernel's double sum `got` of `terms` against fsum: |got - fsum| <= n 2^-52 sum |terms|
    (+ `extra`, the terms' own allowance)."""
    rep = rep or Report(name, EPS["reduction"])
    s, es = fsum(terms)
    n = _t(terms).numel()
    A = float(_t(terms).double().abs().sum())
    unit = max(n * A, 1e-300)
    err = max(abs(float(got) - s) - es - extra, 0.0)
    rep.add(torch.tensor([err / unit if err else 0.0]), (), ("sum",))
    return rep


# ------------------------------------------------------------------------------- points
def quotients(pts, h):
    """p / h in double (exact division of the float32 inputs, one double rounding)."""
    p = _t(pts).double()
    return p / float(np.float32(h))


def _ulp32(q):
    a = q.abs().clamp(min=2.0 ** -126)
    return torch.pow(2.0, torch.floor(torch.log2(a)) - 23)


def cell_candidates(q):
    """Admissible cells (lo, hi) per coordinate of rint(float32(p / h)) (see the module
    docstring); both int64, NaN / inf coordinates give lo > hi."""
    fin = torch.isfinite(q)
    qs = torch.where(fin, q, torch.zeros_like(q))
    exact = qs.float().double() == qs
    e = torch.where(exact, torch.zeros_like(qs), _ulp32(qs))
    lo = torch.round(qs - e).long()                        # torch.round: half to even
    hi = torch.round(qs + e).long()
    lo = torch.where(fin, lo, torch.ones_like(lo))
    hi = torch.where(fin, hi, torch.zeros_like(hi))
    return lo, hi


def check_cell_keys(pts, normals, h, lo, N, keys, unit_normals=None, rep=None, rep_n=None):
    """poisson_cell_keys: keys (n,) int64 against the admissible cells of exact division, and the
    unit normals."""
    rep = rep or Report("cell_keys", 0.0)
    dev = _t(keys).device
    q = quotients(_t(pts, dev), h)
    clo, chi_ = cell_candidates(q)
    lo_t = torch.tensor(lo, device=dev, dtype=torch.int64)
    clo, chi_ = clo - lo_t, chi_ - lo_t
    fin = (clo <= chi_).all(1)
    big = (q.abs() >= 1e9).any(1)                          # the kernel's |q| < 1e9f guard
    must_none = ~fin | big | ((chi_ < 0) | (clo >= N)).any(1)
    may_none = must_none | ((clo < 0) | (chi_ >= N)).any(1)
    nok = torch.ones_like(fin)
    if normals is not None:
        n64 = _t(normals, dev).double()
        L = torch.sqrt((n64 * n64).sum(1))
        nok = (L > 0) & torch.isfinite(L)
        must_none |= ~nok
        may_none |= ~nok
        if unit_normals is not None:
            rep_n = rep_n or Report("cell_keys", EPS["cell_keys"])
            want = torch.where(nok[:, None], n64 / L[:, None], torch.zeros_like(n64))
            got = _t(unit_normals, dev).double()
            need = _need(got, want, want.abs() + 2.0 ** -26)
            need = torch.where(nok[:, None], need, torch.where(got == 0, 0.0, float("inf")))
            rep_n.add(need.amax(1), (0,), ())
    k = _t(keys, dev)
    none = k == KEY_NONE
    kk = torch.where(none, torch.zeros_like(k), k)
    c = torch.stack([kk // (N * N), (kk // N) % N, kk % N], 1)
    inside = ((c >= clo) & (c <= chi_)).all(1)
    bad = torch.where(none, ~may_none, must_none | ~inside)
    rep.mismatch(bad, (0,), ())
    return rep, rep_n


def _hats(q, node, delta):
    """Per axis hat value and its admissible interval of float32 arithmetic."""
    d = (q - node).abs()
    hat = (1 - d).clamp(min=0)
    return hat, (1 - d - delta).clamp(min=0), (1 - d + delta).clamp(min=0, max=1)


def point_weights(qg, lo):
    """Every (point, node) pair of nonzero admissible weight: qg (m,3) the quotients p / h, lo
    the grid's first node.  delta scales with the global |p / h|, whose float32 rounding it
    bounds.  -> list over the 64 corners of (local node (m,3) int64, w64 (m,), err bound (m,),
    mask of the points whose weight there may be nonzero)."""
    delta = U * (qg.abs() + 2) * SAFE
    assert float(delta.max()) < 1, "|p/h| beyond 2^24: the weight bound would be vacuous"
    q = qg - torch.tensor(list(lo), device=qg.device, dtype=torch.float64)
    b = torch.ceil(q - 1 - delta).long()
    out = []
    for dx in range(4):
        for dy in range(4):
            for dz in range(4):
                node = b + torch.tensor([dx, dy, dz], device=q.device)
                hat, lo_, hi_ = _hats(q, node.double(), delta)
                w = hat.prod(1)
                wlo = lo_.prod(1) * (1 - 3 * U)
                whi = hi_.prod(1) * (1 + 3 * U)
                e = torch.maximum(whi - w, w - wlo) * SAFE
                keep = whi > 0
                if bool(keep.any()):
                    out.append((node, w, e, keep))
    return out


def check_splat(pts, nrm, rgb, h, lo, N, V, W, C, wins=None, reps=None):
    """poisson_splat: V, W, C (N^3[,3]) of the points it was given (all with cells in the grid)
    against the float64 hat weights of exact division."""
    reps = reps or {k: Report("splat") for k in ("V", "W", "C")}
    dev = _t(W).device
    p = _t(pts, dev)
    n = _t(nrm, dev).double()
    col = (torch.full_like(n, 255.0) if rgb is None else _t(rgb, dev).double())
    pw = point_weights(quotients(p, h), lo)
    for w in wins or [full(N)]:
        s = [w[a + 3] - w[a] for a in range(3)]
        size = s[0] * s[1] * s[2]
        acc = {k: torch.zeros(size, dtype=torch.float64, device=dev)
               for k in ("W", "eW", "AW", "V0", "V1", "V2", "eV0", "eV1", "eV2", "AV0", "AV1", "AV2",
                         "C0", "C1", "C2", "eC0", "eC1", "eC2")}
        for node, wt, e, keep in pw:
            inw = keep & (node >= torch.tensor(w[:3], device=dev)).all(1) & \
                (node < torch.tensor(w[3:], device=dev)).all(1)
            if not bool(inw.any()):
                continue
            l = node[inw] - torch.tensor(w[:3], device=dev)
            idx = (l[:, 0] * s[1] + l[:, 1]) * s[2] + l[:, 2]
            ww, ee = wt[inw], e[inw]
            acc["W"].index_add_(0, idx, ww)
            acc["eW"].index_add_(0, idx, ee)
            acc["AW"].index_add_(0, idx, ww)
            for a in range(3):
                acc[f"V{a}"].index_add_(0, idx, ww * n[inw, a])
                acc[f"eV{a}"].index_add_(0, idx, ee * n[inw, a].abs())
                acc[f"AV{a}"].index_add_(0, idx, ww * n[inw, a].abs())
                acc[f"C{a}"].index_add_(0, idx, ww * col[inw, a])
                acc[f"eC{a}"].index_add_(0, idx, ee * col[inw, a])
        shp = tuple(s)

        def unit(X, e, A):
            b = e + U * (X.abs() + e) + 2.0 ** -48 * A
            return (b / U).reshape(shp)
        gotW = fetch(W, w[:3], w[3:], dev)
        reps["W"].add(_need(gotW, acc["W"].reshape(shp), unit(acc["W"], acc["eW"], acc["AW"])),
                      w[:3], (0,))
        gv, gc = fetch(V, w[:3], w[3:], dev), fetch(C, w[:3], w[3:], dev)
        nv = torch.stack([_need(gv[..., a], acc[f"V{a}"].reshape(shp),
                                unit(acc[f"V{a}"], acc[f"eV{a}"], acc[f"AV{a}"])) for a in range(3)], -1)
        nc = torch.stack([_need(gc[..., a], acc[f"C{a}"].reshape(shp),
                                unit(acc[f"C{a}"], acc[f"eC{a}"], acc[f"C{a}"])) for a in range(3)], -1)
        reps["V"].add(nv.amax(-1), w[:3], (0,))
        reps["C"].add(nc.amax(-1), w[:3], (0,))
    return reps


def iso_terms(chi, pts, h, lo, N):
    """The kernel's float32 trilinear terms w32 * chi of each point's 8 floor corners (float32
    arithmetic reproduced op for op: one division, floor, one subtraction, two products per
    weight), chi gathered from the (N^3,) field on its device -> (m, 8) float64."""
    chi = _t(chi).reshape(-1)
    dev = chi.device
    p = _t(pts, dev).float()
    q = p / torch.tensor(np.float32(h), device=dev)
    fl = torch.floor(q)
    fr = q - fl
    b = fl.long() - torch.tensor(lo, device=dev)
    out = torch.zeros(len(p), 8, dtype=torch.float64, device=dev)
    for d in range(8):
        dd = ((d >> 2) & 1, (d >> 1) & 1, d & 1)
        w = [fr[:, a] if dd[a] else 1 - fr[:, a] for a in range(3)]
        wt = (w[0] * w[1]) * w[2]
        X = b + torch.tensor(dd, device=dev)
        ok = ((X >= 0) & (X < N)).all(1)
        i = torch.where(ok, (X[:, 0] * N + X[:, 1]) * N + X[:, 2], torch.zeros_like(X[:, 0]))
        out[:, d] = torch.where(ok, wt.double() * chi[i].double(), 0.0)
    return out


def check_iso(chi, pts, h, lo, N, got_sum, rep=None, rep_sum=None):
    """poisson_iso_sum: the sum against fsum of the kernel-rule terms (iso_sum), and each point's
    interpolated chi from exact division against the kernel-rule value (iso; hat weights with
    their bound, chi the kernel's own)."""
    terms = iso_terms(chi, pts, h, lo, N)
    rep_sum = check_reduction(got_sum, terms, rep=rep_sum, name="iso_sum")
    rep = rep or Report("iso")
    chi = _t(chi).reshape(-1)
    dev = chi.device
    qg = quotients(_t(pts, dev), h)
    v64 = torch.zeros(len(qg), dtype=torch.float64, device=dev)
    ev = torch.zeros_like(v64)
    for node, wt, e, keep in point_weights(qg, lo):
        ok = keep & ((node >= 0) & (node < N)).all(1)
        i = torch.where(ok, (node[:, 0] * N + node[:, 1]) * N + node[:, 2], torch.zeros_like(node[:, 0]))
        c = torch.where(ok, chi[i].double(), 0.0)
        v64 += wt * c
        ev += e * c.abs()
    v32 = terms.sum(1)
    A = terms.abs().sum(1)
    unit = (ev + 2.0 ** -48 * A) / U
    rep.add(_need(v32, v64, unit), (0,), ())
    return rep, rep_sum


def check_moments(pts, start, centre, mom, rep=None):
    """poisson_cell_moments: (nc, 10) double moments of d = p - centre per cell."""
    rep = rep or Report("moments")
    dev = _t(mom).device
    st = _t(start, dev).long()
    cnt = st[1:] - st[:-1]
    cell = torch.repeat_interleave(torch.arange(len(cnt), device=dev), cnt)
    p = _t(pts, dev).double()[:int(st[-1])]
    d = p - torch.tensor(list(centre), device=dev, dtype=torch.float64)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    t = torch.stack([torch.ones_like(x), x, y, z, x * x, x * y, x * z, y * y, y * z, z * z], 1)
    ref = torch.zeros(len(cnt), 10, dtype=torch.float64, device=dev).index_add_(0, cell, t)
    A = torch.zeros_like(ref).index_add_(0, cell, t.abs())
    got = _t(mom, dev).double()
    rep.add(_need(got, ref, A * cnt[:, None].double().clamp(min=1)).amax(1), (0,), ())
    return rep


def block_moments(ckeys, mom, N):
    """Sum of the moments of the 3x3x3 cells around each cell (x-major), float64."""
    k = _t(ckeys).long()
    dev = k.device
    m = _t(mom, dev).double()
    x, y, z = k // (N * N), (k // N) % N, k % N
    out = torch.zeros_like(m)
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dz in (-1, 0, 1):
                X, Y, Z = x + dx, y + dy, z + dz
                ok = (X >= 0) & (Y >= 0) & (Z >= 0) & (X < N) & (Y < N) & (Z < N)
                kk = (X * N + Y) * N + Z
                j = torch.searchsorted(k, kk).clamp(max=len(k) - 1)
                hit = ok & (k[j] == kk)
                out += torch.where(hit[:, None], m[j], 0.0)
    return out


def check_normals(ckeys, mom, N, cn, cok, rep=None, exempt_cap=None):
    """poisson_cell_normals against np.linalg.eigh of the block covariance."""
    rep = rep or Report("normals")
    M = block_moments(ckeys, mom, N).cpu().numpy()
    got = _t(cn).double().cpu().numpy()
    gok = _t(cok).cpu().numpy().astype(bool)
    m0 = M[:, 0]
    few = m0 < 3
    with np.errstate(all="ignore"):
        mu = M[:, 1:4] / m0[:, None]
        cov = np.empty((len(M), 3, 3))
        idx = [(0, 0, 4), (0, 1, 5), (0, 2, 6), (1, 1, 7), (1, 2, 8), (2, 2, 9)]
        for a, b, j in idx:
            cov[:, a, b] = cov[:, b, a] = M[:, j] / m0 - mu[:, a] * mu[:, b]
        S = (M[:, 4] + M[:, 7] + M[:, 9]) / m0
    cov[few] = np.eye(3)
    S[few] = 1.0
    lam, vec = np.linalg.eigh(cov)
    band = K_EIG * 2.0 ** -52 * S
    ok64 = (lam[:, 2] > 0) & (lam[:, 1] > RANK_EPS * lam[:, 2])
    amb = (np.abs(lam[:, 1] - RANK_EPS * lam[:, 2]) <= band) | (np.abs(lam[:, 2]) <= band)
    bad_ok = np.where(few, gok, (gok != ok64) & ~amb)
    zero_bad = ~gok & (got != 0).any(1)
    rep.mismatch(torch.from_numpy(bad_ok | zero_bad), (0,), ())
    gap = lam[:, 1] - lam[:, 0]
    v0 = vec[:, :, 0]
    sel = gok & ~few
    exempt = sel & (gap <= GAP_FLOOR * S)
    chk = sel & ~exempt
    L = np.linalg.norm(got, axis=1)
    sinang = np.linalg.norm(np.cross(got, v0), axis=1) / np.where(L > 0, L, 1)
    need = np.where(chk, sinang * np.maximum(gap, 0) / S, 0.0)
    need = np.where(chk & (np.abs(L - 1) > 1e-12), np.inf, need)
    rep.add(torch.from_numpy(need), (0,), ())
    rep.exempt += int(exempt.sum())
    return rep


def check_orient(pts, pcell, cn, cams, out, rep=None):
    """poisson_orient: float32(+-cn) toward the nearest camera (ties to the lower index)."""
    rep = rep or Report("orient")
    dev = _t(out).device
    p = _t(pts, dev).float().double()
    cams = _t(np.asarray(cams, np.float64), dev).double().reshape(-1, 3)
    d = p[:, None, :] - cams[None]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    best = d2.min(1).values
    first = torch.argmin(torch.where(d2 == best[:, None], torch.arange(len(cams), device=dev)[None].double(),
                                     float("inf")), 1)
    near = d2 <= best[:, None] * (1 + 4 * 2.0 ** -52)
    exact_tie = (d2 == best[:, None]).sum(1) > 1
    n = _t(cn, dev).double()[_t(pcell, dev).long()]
    got = _t(out, dev).double()
    plus = n.float().double()
    can_p = torch.zeros(len(p), dtype=torch.bool, device=dev)
    can_m = torch.zeros_like(can_p)
    for k in range(len(cams)):
        # an exact tie goes to its lower index; cameras merely near the best stay admissible
        allowed = torch.where(exact_tie, (first == k) | (near[:, k] & (d2[:, k] != best)), near[:, k])
        t = n * (cams[k][None] - p)
        dot = t.sum(1)
        mag = t.abs().sum(1) * 4 * 2.0 ** -52
        can_p |= allowed & (dot >= -mag)
        can_m |= allowed & (dot < mag)
    okp = (got == plus).all(1)
    okm = (got == -plus).all(1)
    rep.mismatch(~((okp & can_p) | (okm & can_m)), (0,), ())
    return rep


# ------------------------------------------------------------------------------- trim and bricks
def box5(a):
    """5x5x5 sum over the inner part of a box padded by 2 (first three axes)."""
    for ax in range(3):
        n = a.shape[ax] - 4
        a = sum(a.narrow(ax, d, n) for d in range(5))
    return a


def check_trim(W, keep, N, wins=None, rep=None):
    rep = rep or Report("trim")
    for w in wins or [full(N)]:
        dev = _t(keep).device
        lo, hi = _pad(w, 2)
        P = (fetch(W, lo, hi, dev) > 0).double()
        for ax in range(3):
            n = P.shape[ax] - 4
            m = P.narrow(ax, 0, n)
            for d in range(1, 5):
                m = torch.maximum(m, P.narrow(ax, d, n))
            P = m
        got = fetch(keep, w[:3], w[3:], dev)
        rep.mismatch((got != 0) != (P > 0), w[:3], (0,))
    return rep


def check_brick_flags(keep, N, lo, b0, nb, flags, rep=None):
    rep = rep or Report("brick_flags")
    k = _t(keep).reshape(N, N, N)
    dev = k.device
    o = [lo[a] - 8 * b0[a] for a in range(3)]
    P = torch.zeros(8 * nb[0], 8 * nb[1], 8 * nb[2], dtype=torch.uint8, device=dev)
    P[o[0]:o[0] + N, o[1]:o[1] + N, o[2]:o[2] + N] = (k != 0).to(torch.uint8)
    ref = P.reshape(nb[0], 8, nb[1], 8, nb[2], 8).amax((1, 3, 5))
    del P
    rep.mismatch((_t(flags, dev).reshape(ref.shape) != 0) != (ref != 0), (0, 0, 0), ())
    return rep


def voxel_nodes(keys, lo):
    """Local node (nb*512, 3) of every brick voxel of mesh.cu's layout."""
    k = _t(keys).long()
    dev = k.device
    B = 1 << 20
    b = torch.stack([(k >> 42) - B, ((k >> 21) & 0x1FFFFF) - B, (k & 0x1FFFFF) - B], 1)
    l = torch.arange(512, device=dev)
    off = torch.stack([l & 7, (l >> 3) & 7, l >> 6], 1)
    g = (b[:, None, :] * 8 + off[None]).reshape(-1, 3)
    return g - torch.tensor(list(lo), device=dev)


def check_fill(keys, keep, W, C, chi, iso, weight, color, tsdf, N, lo, wins=None, reps=None):
    """poisson_fill_bricks and poisson_fill_tsdf over the voxels whose node lies in a window;
    voxels outside the grid (any window) must have weight 0, colour 0 and tsdf 0."""
    reps = reps or dict(fill_bricks=Report("fill_bricks"), fill_tsdf=Report("fill_tsdf"))
    g = voxel_nodes(keys, lo)
    dev = g.device
    wt = _t(weight, dev).reshape(-1)
    col = _t(color, dev).reshape(-1, 3).double()
    ts = _t(tsdf, dev).reshape(-1).double()
    outside = ~((g >= 0) & (g < N)).all(1)
    reps["fill_bricks"].mismatch((outside & ((wt != 0) | (col != 0).any(1))), (0,), ("voxel",))
    reps["fill_tsdf"].mismatch(outside & (ts != 0), (0,), ("voxel",))
    for w in wins or [full(N)]:
        inw = ((g >= torch.tensor(w[:3], device=dev)) & (g < torch.tensor(w[3:], device=dev))).all(1)
        if not bool(inw.any()):
            continue
        l = g[inw] - torch.tensor(w[:3], device=dev)
        lo2, hi2 = _pad(w, 2)
        Wb = box5(fetch(W, lo2, hi2, dev))
        Cb = box5(fetch(C, lo2, hi2, dev))
        K = fetch(keep, w[:3], w[3:], dev) != 0
        X = fetch(chi, w[:3], w[3:], dev)
        sel = (l[:, 0], l[:, 1], l[:, 2])
        kept = K[sel]
        with torch.no_grad():
            ref = torch.where(kept[:, None], Cb[sel] / Wb[sel][:, None], 0.0)
        gw, gc = wt[inw], col[inw]
        bad_w = gw != kept.float()
        need = _need(gc, ref, ref.abs()).amax(1)
        need = torch.where(bad_w, float("inf"), need)
        reps["fill_bricks"].add(need, (0,), ("voxel",))
        x = X[sel]
        tref = torch.where(gw > 0, x - iso, 0.0)
        unit = tref.abs() + 2.0 ** -28 * (x.abs() + abs(iso))
        reps["fill_tsdf"].add(_need(ts[inw], tref, unit), (0,), ("voxel",))
    return reps


# ------------------------------------------------------------------------------- float64 solve
def laplacian(x, h):
    """(N^3) float64 field -> L x at the finest interior, 0 on the outer layer (torch)."""
    n = x.shape[0]
    s = torch.zeros_like(x)
    i = slice(1, -1)
    s[i, i, i] = ((((x[:-2, i, i] + x[2:, i, i]) + x[i, :-2, i]) + x[i, 2:, i]) + x[i, i, :-2]) + x[i, i, 2:]
    s[i, i, i] -= 6 * x[i, i, i]
    return s / (h * h)


def _ref_smooth(e, r, level, h, sweeps):
    n = e.shape[0]
    P = torch.zeros(n + 2, n + 2, n + 2, dtype=torch.float64, device=e.device)
    P[1:-1, 1:-1, 1:-1] = e
    w = full(n)
    inner = interior(w, n, level, e.device)
    x, y, z = _grid_xyz(w, e.device)
    par = (x + y + z) % 2
    for _ in range(sweeps):
        for parity in (0, 1):
            s, _a = _nbs(P)
            m = inner & (par == parity)
            P[1:-1, 1:-1, 1:-1] = torch.where(m, (s - h * h * r) / 6, P[1:-1, 1:-1, 1:-1])
    return P[1:-1, 1:-1, 1:-1].clone()


def _ref_mg_residual(e, r, level, h):
    n = e.shape[0]
    P = torch.zeros(n + 2, n + 2, n + 2, dtype=torch.float64, device=e.device)
    P[1:-1, 1:-1, 1:-1] = e
    s, _a = _nbs(P)
    out = r - (s - 6 * e) / (h * h)
    return torch.where(interior(full(n), n, level, e.device), out, 0.0)


def _ref_restrict(f):
    nf = f.shape[0]
    nc = nf // 2
    F = torch.zeros(nf + 1, nf + 1, nf + 1, dtype=torch.float64, device=f.device)
    F[1:, 1:, 1:] = f
    Ms = [_restrict_matrix(0, nc, -1, nf, nc, f.device)] * 3
    return _apply3(Ms, F)


def _ref_prolong(c):
    nc = c.shape[0]
    C = torch.zeros(nc + 1, nc + 1, nc + 1, dtype=torch.float64, device=c.device)
    C[:nc, :nc, :nc] = c
    Ms = [_prolong_matrix(0, 2 * nc, 0, nc + 1, c.device)] * 3
    return _apply3(Ms, C)


def vcycle64(r, h, level=0, pre=2, post=2, coarse_sweeps=50):
    """The kernels' V(2,2) cycle (same levels, rules and sweep order) in float64."""
    n = r.shape[0]
    if n <= COARSEST:
        return _ref_smooth(torch.zeros_like(r), r, level, h, coarse_sweeps)
    e = _ref_smooth(torch.zeros_like(r), r, level, h, pre)
    res = _ref_mg_residual(e, r, level, h)
    ec = vcycle64(_ref_restrict(res), float(np.float32(2 * h)), level + 1, pre, post, coarse_sweeps)
    e = e + torch.where(interior(full(n), n, level, r.device), _ref_prolong(ec), 0.0)
    return _ref_smooth(e, r, level, h, post)


def multigrid64(b, h, tol=1e-5, max_cycles=40):
    """float64 multigrid of the kernels' rule on b (N^3 torch) -> (chi, per-cycle ratios)."""
    b = b.double()
    h = float(np.float32(h))
    chi = torch.zeros_like(b)
    bn = float(torch.linalg.vector_norm(b))
    ratios = []
    while True:
        r = b - laplacian(chi, h)
        r = torch.where(interior(full(b.shape[0]), b.shape[0], 0, b.device), r, 0.0)
        ratios.append(float(torch.linalg.vector_norm(r)) / bn)
        if ratios[-1] <= tol or len(ratios) > max_cycles:
            return chi, ratios
        chi = chi + vcycle64(r, h)


# ------------------------------------------------------------------------------- edge clouds
def tie_cloud(depth, n=2000, seed=0):
    """A sphere of radius 0.8 inside two corner anchors that make h = float32(1.1 E / N) exactly
    2^(1 - depth), plus points whose quotient p / h is an exact tie k + 1/2 (k even and odd) or an
    exact integer, verified in float32 and in float64 -> (points, normals, tie mask)."""
    from oracle import poisson_oracle as O
    N = 1 << depth
    target = np.float32(2.0 / N)
    a = np.float32(1 / 1.1)
    for _ in range(64):
        h = np.float32(1.1 * (2 * np.float64(a)) / N)
        if h == target:
            break
        a = np.nextafter(a, np.float32(2 if h < target else 0))
    assert h == target
    p, nrm = O.sphere(n, radius=0.8, seed=seed, noise=0.005)
    rng = np.random.default_rng(seed)
    k = rng.integers(-20, 20, (600, 3)).astype(np.float32)
    t = k + np.where(rng.random((600, 3)) < 0.6, np.float32(0.5), np.float32(0))
    q = (t * h).astype(np.float32)
    assert ((q / h).astype(np.float32) == t).all() and ((q.astype(np.float64) / float(h)) == t).all()
    anchors = np.array([[-a, -a, -a], [a, a, a]], np.float32)
    pts = np.concatenate([p, q, anchors]).astype(np.float32)
    u = rng.normal(size=(len(q) + 2, 3))
    nn = np.concatenate([nrm, (u / np.linalg.norm(u, axis=1, keepdims=True)).astype(np.float32)])
    tie = np.r_[np.zeros(len(p), bool), (np.abs(t - np.floor(t)) == 0.5).any(1), np.zeros(2, bool)]
    return pts, nn, tie


CONTRACTION = 1.25


def contraction_ok(got, want, factor=CONTRACTION):
    """Per-cycle convergence: got and want are ||r|| / ||b|| before each cycle and at the end.
    Every cycle's contraction got[k] / got[k-1] must be within `factor` of the float64 cycle's,
    and the cycle counts within 1."""
    if abs(len(got) - len(want)) > 1:
        return False
    for k in range(1, min(len(got), len(want))):
        if got[k] / got[k - 1] > factor * (want[k] / want[k - 1]):
            return False
    return True


def hs_levels(h, N):
    """The per-level spacings poisson.py passes: float32(h 2^l) for each level down to 8."""
    return [float(np.float32(h * (1 << l))) for l in range(32) if (N >> l) >= COARSEST]
