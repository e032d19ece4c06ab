"""The float64 fusion reference (oracle/fusion_fp64.py) on the CPU:

  * pinned to oracle/fusion_oracle.py (itself pinned to the reference's functions) on the
    golden 64x48 fixture: every unambiguous mask decision equal, every reprojection and warped
    colour within the admissible bound;
  * an fp32 restatement of geo_fuse_kernel, in the kernel's operation order, passes every check
    with no exception at 320x256 with 10 and 16 sources and on the known-answer edge cases;
  * the same restatement with one injected defect fails, and the report names a (source, y, x)
    where the defect changed an output;
  * the share of ambiguous mask decisions on a 1152x864 scene stays under AMBIGUOUS_MAX.
"""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import synth_scenes
from oracle import fusion_fp64 as FF
from oracle import fusion_oracle as FO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# Share of (source, pixel) mask decisions the bounds leave open on the 1152x864 scene: 5.9e-4
# (it depends only on the oracle and the data); the ceiling is the power of two above twice that.
AMBIGUOUS_MAX = 2.0 ** -9


# ------------------------------------------------------------------------------- restatement
def restate(inp, defect=None):
    """geo_fuse_kernel in torch float32 (CPU), one rounding per operation in the kernel's order,
    with an optional injected defect."""
    d = inp["depth_ref"].float()
    H, W = d.shape
    S = len(inp["depth_srcs"])
    y, x = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32),
                          indexing="ij")
    rs = np.asarray(inp["rs"], np.float32).reshape(-1, 12)
    sr = np.asarray(inp["sr"], np.float32).reshape(-1, 12)
    img_ref = inp.get("image_ref")
    use_img = img_ref is not None and inp.get("image_srcs") is not None
    dsum = d.clone()
    csum = img_ref.float().clone() if img_ref is not None else torch.zeros(H, W, 3)
    cnt = torch.zeros(H, W, dtype=torch.int32)
    masks = torch.zeros(S, H, W, dtype=torch.bool)
    reproj = torch.zeros(S, H, W)
    f = lambda v: torch.tensor(float(v), dtype=torch.float32)

    def row(a, v):
        return ((f(a[0]) * v[0] + f(a[1]) * v[1]) + f(a[2]) * v[2]) + f(a[3])

    def sample(img, ix, iy, fx, fy):
        if img.dim() == 2:
            img = img.unsqueeze(-1)
            squeeze = True
        else:
            squeeze = False

        def tap(xx, yy):
            ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
            v = img[yy.clamp(0, H - 1), xx.clamp(0, W - 1)]
            if defect == "border_clamp":
                return v
            return torch.where(ok.unsqueeze(-1), v, torch.zeros_like(v))
        one = torch.tensor(1.0)
        w00, w01 = ((one - fx) * (one - fy)).unsqueeze(-1), (fx * (one - fy)).unsqueeze(-1)
        w10, w11 = ((one - fx) * fy).unsqueeze(-1), (fx * fy).unsqueeze(-1)
        out = ((tap(ix, iy) * w00 + tap(ix + 1, iy) * w01) + tap(ix, iy + 1) * w10) + tap(ix + 1, iy + 1) * w11
        return out[..., 0] if squeeze else out

    for s in range(S):
        if defect == "skip_last" and s == S - 1:
            continue
        A, B = rs[s], sr[s]
        if defect == "swap" and s == 1:
            A, B = B, A
        X, Y = x * d, y * d
        qx, qy, qz = row(A[0:4], (X, Y, d)), row(A[4:8], (X, Y, d)), row(A[8:12], (X, Y, d))
        xs, ys = qx / qz, qy / qz
        fin = torch.isfinite(xs) & torch.isfinite(ys)
        with torch.no_grad():
            t = torch.where(fin, xs, torch.zeros_like(xs)) * 32
            u = torch.where(fin, ys, torch.zeros_like(ys)) * 32
            rnd = torch.floor if defect == "floor_bin" else torch.round
            sx = rnd(t.double()).clamp(-2.0 ** 31, 2.0 ** 31 - 1).long()
            sy = rnd(u.double()).clamp(-2.0 ** 31, 2.0 ** 31 - 1).long()
        mode = "trunc" if defect == "trunc_div" else "floor"
        ix, iy = torch.div(sx, 32, rounding_mode=mode), torch.div(sy, 32, rounding_mode=mode)
        fx, fy = (sx & 31).float() * (1 / 32), (sy & 31).float() * (1 / 32)
        ds = torch.where(fin, sample(inp["depth_srcs"][s].float(), ix, iy, fx, fy), torch.zeros_like(d))
        col = torch.zeros(H, W, 3)
        if use_img:
            col = torch.where(fin.unsqueeze(-1), sample(inp["image_srcs"][s].float(), ix, iy, fx, fy), col)
        U, V = xs * ds, ys * ds
        rx, ry, rz = row(B[0:4], (U, V, ds)), row(B[4:8], (U, V, ds)), row(B[8:12], (U, V, ds))
        dx, dy = rx / rz - x, ry / rz - y
        p = dx * dx + dy * dy
        m_pix = p <= 1 if defect == "le_pixel" else p < 1
        m_dep = ((rz - d) / (ds if defect == "div_ds" else d)).abs() < f(0.01)
        m = m_pix & m_dep
        dsum = dsum + torch.where(m, rz, torch.zeros_like(rz))
        csum = csum + torch.where(m.unsqueeze(-1), col, torch.zeros_like(col))
        cnt += m.int()
        masks[s] = m
        reproj[s] = torch.where(m, rz, torch.zeros_like(rz))
    n1 = (cnt + 1).float()
    inv = 1 / n1
    dref = dsum / n1
    image_refined = None
    if img_ref is not None:
        image_refined = csum / cnt.float().unsqueeze(-1) if defect == "image_div_cnt" else csum * inv.unsqueeze(-1)
    keep = cnt >= int(inp["min_consistent"])
    if inp.get("proba_ref") is not None:
        keep = keep & (upsample4_fp32(inp["proba_ref"].float(), H, W, defect == "align_corners")
                       > f(inp["conf"]))
    M = np.asarray(inp["ref2world"], np.float32).reshape(-1)
    Xr, Yr = x * dref, y * dref
    points = torch.stack([row(M[4 * r:4 * r + 4], (Xr, Yr, dref)) for r in range(3)], -1)
    return dict(mask=masks, reproj=reproj, geo_count=cnt, mask_final=keep, depth_refined=dref,
                image_refined=image_refined, points=points)


def upsample4_fp32(p, H, W, align_corners=False):
    h4, w4 = p.shape

    def coords(n, n_in):
        i = torch.arange(n, dtype=torch.float64)
        f = i * (n_in - 1) / (n - 1) if align_corners else (i + 0.5) * 0.25 - 0.5
        f = f.float()
        s = torch.floor(f)
        f = f - s
        s = s.long()
        lo, hi = s < 0, s >= n_in - 1
        f = torch.where(lo | hi, torch.zeros_like(f), f)
        s = torch.where(lo, 0, torch.where(hi, n_in - 1, s))
        return s, (s + 1).clamp(max=n_in - 1), f
    x0, x1, fx = coords(W, w4)
    y0, y1, fy = coords(H, h4)
    one = torch.tensor(1.0)
    r0 = p[y0][:, x0] * (one - fx) + p[y0][:, x1] * fx
    r1 = p[y1][:, x0] * (one - fx) + p[y1][:, x1] * fx
    return r0 * (one - fy)[:, None] + r1 * fy[:, None]


# ------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def g():
    with np.load(os.path.join(ROOT, "tests", "golden", "fusion_64x48.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def scene16():
    views = synth_scenes.sphere_scene(17, (320, 256), seed=3, radius=150)
    return FF.scene_inputs(views, 16, seed=3)


def _check(tag, inp, out, exact=False):
    rep = FF.check_fuse(inp, out, exact=exact)
    print(f"[fp64] {tag}{' exact' if exact else ''}: {rep.describe()}")
    return rep


# ------------------------------------------------------------------------------- tests
def test_oracle_matches_fusion_oracle_golden(g):
    """fusion_oracle (numpy float32 + cv2) on the golden fixture lies in the admissible sets."""
    H, W = g["depths"][0].shape
    d_ref = torch.from_numpy(g["depths"][0])
    amb = 0
    for s in range(1, len(g["P"])):
        r, m, i2 = FO.check_geo_consistency(g["depths"][0], g["P"][0], g["depths"][s], g["P"][s],
                                            g["images"][0], g["images"][s], (W, H))
        ref = FF.source_ref(d_ref, torch.from_numpy(g["depths"][s]), torch.from_numpy(g["images"][s]),
                            FF.rel(g["P"][s], g["P"][0]), FF.rel(g["P"][0], g["P"][s]),
                            reproj=torch.from_numpy(r))
        ct, cf = ref["can_true"].numpy(), ref["can_false"].numpy()
        amb += int((ct & cf).sum())
        assert not (m & ~ct).any() and not (~m & ~cf).any(), f"source {s}: mask outside the set"
        assert (ref["rz_ratio"].numpy()[m] <= 1).all(), f"source {s}: reprojection outside its bound"
        lo, hi = ref["col_lo"].numpy(), ref["col_hi"].numpy()
        mm = m[..., None]
        assert ((i2 >= lo) | ~mm).all() and ((i2 <= hi) | ~mm).all(), f"source {s}: colour out of bound"
        print(f"[fp64] golden source {s}: {int(m.sum())} consistent, {int((ct & cf).sum())} ambiguous")
    up, e = FF.upsample4_ref(torch.from_numpy(g["proba"]))
    assert ((torch.from_numpy(FO.resize4_linear(g["proba"])).double() - up).abs() <= e).all()
    assert ((torch.from_numpy(g["proba_up"]).double() - up).abs() <= e).all()


@pytest.mark.parametrize("S", [10, 16])
def test_restatement_passes(scene16, S):
    inp = dict(scene16)
    inp["depth_srcs"], inp["image_srcs"] = inp["depth_srcs"][:S], inp["image_srcs"][:S]
    inp["rs"], inp["sr"] = inp["rs"][:S], inp["sr"][:S]
    rep = _check(f"restated S={S}", inp, restate(inp))
    assert rep.ok, rep.describe()
    pairs = rep.pairs
    assert rep.certain_true > 0.02 * pairs and rep.certain_false > 0.2 * pairs, rep.describe()


@pytest.mark.parametrize("name", [c[0] for c in FF.edge_cases()])
def test_restatement_edge_cases(name):
    inp = dict(FF.edge_cases())[name]
    out = restate(inp)
    for exact in (True, False):
        rep = _check(f"restated {name}", inp, out, exact)
        assert rep.ok, rep.describe()
    if name == "confidence":
        mf = out["mask_final"]
        for (r, c), want in FF.CONF_CORNERS.items():
            assert bool(mf[14 * r:14 * r + 2, 14 * c:14 * c + 2].all() if want
                        else ~mf[14 * r:14 * r + 2, 14 * c:14 * c + 2].any())


DEFECTS = ["border_clamp", "trunc_div", "floor_bin", "le_pixel", "div_ds", "skip_last", "swap",
           "align_corners", "image_div_cnt"]


def _changed(good, bad, loc):
    """Did the defect change an output at loc ((s, y, x) or (y, x))?"""
    if len(loc) == 3:
        s, yy, xx = loc
        return bool(good["mask"][s, yy, xx] != bad["mask"][s, yy, xx]
                    or good["reproj"][s, yy, xx] != bad["reproj"][s, yy, xx])
    yy, xx = loc
    return any(not torch.equal(good[k][yy, xx], bad[k][yy, xx])
               for k in ("mask_final", "depth_refined", "image_refined", "geo_count")
               if good[k] is not None)


@pytest.mark.parametrize("defect", DEFECTS)
def test_injected_defect_fails(scene16, defect):
    inp = dict(scene16)
    S = 10
    inp["depth_srcs"], inp["image_srcs"] = inp["depth_srcs"][:S], inp["image_srcs"][:S]
    inp["rs"], inp["sr"] = inp["rs"][:S], inp["sr"][:S]
    cases = [("scene", inp)] + FF.edge_cases()
    caught = []
    for name, case in cases:
        good, bad = restate(case), restate(case, defect)
        for exact in ((False,) if name == "scene" else (True, False)):
            rep = FF.check_fuse(case, bad, exact=exact)
            if rep.ok:
                continue
            what, loc = rep.first_failure()
            assert _changed(good, bad, loc), f"{defect}: {name} reports {what} at {loc}, unchanged there"
            caught.append((name, exact, what, loc))
    print(f"[fp64] defect {defect}: caught by {caught}")
    assert caught, f"{defect} passes every check"


def test_ambiguous_fraction_1152x864():
    views = synth_scenes.sphere_scene(5, (1152, 864), seed=11, radius=150)
    inp = FF.scene_inputs(views, 4, seed=11)
    amb = pairs = unc = 0
    for s in range(4):
        ref = FF.source_ref(inp["depth_ref"], inp["depth_srcs"][s], None, inp["rs"][s], inp["sr"][s])
        amb += int((ref["can_true"] & ref["can_false"]).sum())
        unc += int(ref["unconstrained"].sum())
        pairs += ref["can_true"].numel()
    print(f"[fp64] 1152x864 S=4: {amb} ambiguous of {pairs} mask decisions ({amb / pairs:.2e}), "
          f"{unc} unconstrained")
    assert amb <= AMBIGUOUS_MAX * pairs
