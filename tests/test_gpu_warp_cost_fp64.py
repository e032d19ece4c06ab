"""Every K1 kernel and the K1 backward element by element against the float64 reference
(oracle/warp_cost_fp64.py):

  * the production stages through the entry points the cascade calls: cfg2 / cfg3 (640x512,
    V=3, G=1 / 8) at all three levels through warp_cost_ladder in its three hypothesis forms,
    TF32-rounded and blocked as well as channels-last fp32; cfg4 (1152x864, V=5) and cfg5
    (1920x1056, V=7) through ops.warp_cost with the materialised hypotheses;
  * the inverse-depth sweep (README "Wide depth ranges") through the same entry point: the cfg2 /
    cfg3 stages with a float u_near, per-item (B,) first and step and a (B, h, w) first map, and
    the staging geometries at 1 and 2 source views, C in {8, 16, 32}, G in {1, 8}, among them
    two asserted by construction on the CPU (INV_EDGES): inverse-wide (far / near >= 10, a pair
    of near planes already spans more than the staged box, so stage_boxes halves its runs) and
    inverse-behind (part of the near sweep has q_z <= 1e-7).  The oracle's hypotheses come from
    INV.ladder_f32, which Ladder.materialize() must equal bit for bit;
  * every instantiation: the 48 TMA-staged kernels (24 uniform, 24 inverse), the 68 gather kernels (1, 2, 4, 6 source
    views x C in {8, 16, 32, other} x variance / group-wise x NCHW / NHWC output, plus the
    generic run-time-V kernel), both homo_warp kernels and the NCHW-feature transpose, at
    ragged shapes, h or w = 2, D = 1, odd D and D not a multiple of the depth chunk, under
    default and stress poses, wide sweeps, depth discontinuities inside a tile, non-monotone
    hypotheses, hypotheses clamped to 1e-7 near the camera and integer / half-integer
    translations that put samples exactly on the image border and on texel centres;
  * a coverage test that runs the whole table under torch.profiler and asserts that every
    instantiation above was launched;
  * the TF32 stores: the rounded output of every kernel equals tf32_rna of the same call's
    unrounded output, bit for bit;
  * casmvs_warp_cost_bwd at the 640x512 training crop and at 4 and 15 source views.

Features are N(0, 1), unsmoothed; B = 2 with per-item features, projections and hypotheses.
EPS holds, per kernel family, at most 4x the worst eps needed over this file on an H100 and never
more than EPS_CEIL; LOOSE_CEIL the loose share (bound above 1 % of the magnitude) likewise."""
import os
import re
import subprocess
import sys
import zlib

import pytest
import torch

from casmvsnet_pl_b200 import _lib, ops, synth
from oracle import inverse_depth_fp64 as INV
from oracle import warp_cost_fp64 as W

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

EPS_CEIL = {"staged": 2.0 ** -17, "gather": 2.0 ** -17, "homo": 2.0 ** -17, "bwd": 2.0 ** -14}
LOOSE_CEIL_MAX = 0.1
# Worst eps needed over every case of this file (it prints them), measured on an H100 80GB HBM3
# at a 400 W power limit; each eps is the largest power of two within 4x of it.  homo_warp needed
# none (the blend term of the bound covers its arithmetic): its eps is a nominal 2^-24.
EPS = {
    "staged": 2.0 ** -22,        # TMA-staged kernels (warp_cost_smem.cu): 1.05e-7
    "gather": 2.0 ** -21,        # gather kernels (warp_cost.cu): 1.57e-7
    "homo": 2.0 ** -24,          # homo_warp: 0
    "bwd": 2.0 ** -22,           # casmvs_warp_cost_bwd, per magnitude of the scattered terms: 8.9e-8
}
# Loose share (bound above 1 % of the element's texel-scale magnitude), worst over the file on the
# same H100: forward 9.6e-5 (samples on the image border), backward 2.6e-2 (stress poses: texels
# reached by samples next to q_z = 0, whose landing texel the bound cannot pin down).
LOOSE_CEIL = {"cost": 2.0 ** -12, "bwd": 2.0 ** -4}


def _seed(name):
    return zlib.crc32(name.encode())


# ------------------------------------------------------------------------------- inputs
def _proj(pose, V, W_, H, level, B):
    """(B, V-1, 3, 4) on DEV, distinct per batch item.  grid: pure translations u = x + a + T/d
    (q_z = 1) that with hypotheses 1, 2, 4 put samples exactly on x = -1, 0, w-1, w and on texel
    centres and midpoints."""
    if pose == "grid":
        P = torch.zeros(B, V - 1, 3, 4)
        P[..., 0, 0] = P[..., 1, 1] = P[..., 2, 2] = 1
        for v in range(V - 1):
            a, T = ((-1.0, 2.0), (0.0, -2.0), (0.5, 1.0), (-0.5, 0.0))[v % 4]
            P[:, v, 0, 2], P[:, v, 0, 3] = a, T
            P[:, v, 1, 2] = (0.0, 0.5, -1.0, 1.0)[v % 4]
            P[:, v, 1, 3] = (0.0, 2.0, 0.0, -2.0)[v % 4]
        for b in range(B):
            P[b, :, 0, 2] += b
        return P.to(DEV)
    stress = pose == "stress"
    P = synth.projection_matrices(V, W_, H, stress=stress, behind_view=1 if stress else None)
    P = P[:, level].unsqueeze(0).repeat(B, 1, 1, 1)
    for b in range(1, B):
        P[b, :, 0, 2] += 1.37 * b
        P[b, :, 1, 2] -= 0.71 * b
    return P.to(DEV)


def _feats(g, B, V, C, h, w, nchw=False):
    """Logical (B, V, C, h, w) N(0,1) features, channels-last storage (or contiguous NCHW)."""
    f = torch.randn(B, V, h, w, C, generator=g, device=DEV)
    f = f.permute(0, 1, 4, 2, 3)
    return f.contiguous() if nchw else f


def _first_map(g, B, h, w, D, step, kind):
    """Per-pixel first rung, like get_depth_values after the upsampled depth of the previous
    stage: a smooth field around 600 (distinct per batch item) minus D/2 steps.  clamped: a patch
    clamped to 1e-7 (the near-camera rule); disc: a depth step inside the pixel tiles."""
    ys = torch.arange(h, device=DEV, dtype=torch.float32).view(1, h, 1)
    xs = torch.arange(w, device=DEV, dtype=torch.float32).view(1, 1, w)
    bb = torch.arange(B, device=DEV, dtype=torch.float32).view(B, 1, 1)
    depth = 600.0 + 25.0 * torch.sin(xs / 23.0 + bb) * torch.cos(ys / 17.0) + 9.0 * bb
    depth = depth + torch.rand(B, h, w, generator=g, device=DEV)
    if kind == "disc":
        depth = depth - 150.0 * (xs > w // 3 + 0.5) + 80.0 * (ys > h // 2 + 0.5)
    first = (depth - D / 2 * step).clamp_min(1e-7)
    if kind == "clamped":
        first[:, : max(1, h // 5), : max(1, w // 4)] = 1e-7
    return first.contiguous()


# near / far depth of the inverse ladders: the DTU range of synth.make_inputs; wide: a ratio of
# 12 whose near plane still lands in the source image while one plane step of a short sweep
# moves a sample by more than a staged box; behind: a ratio of 12 across the depth (about 600)
# where the behind_view camera's q_z changes sign (INV_EDGES)
_INV_RANGE = {"dtu": (synth.DEPTH_MIN, synth.DEPTH_MIN + 47 * 4 * synth.DEPTH_INTERVAL),
              "wide": (90.0, 1080.0), "behind": (300.0, 3600.0)}
assert _INV_RANGE["wide"][1] >= 10 * _INV_RANGE["wide"][0]


def _inv_ladder(g, kind, B, D, h, w, level):
    """An inverse ops.Ladder (first and step in 1/depth): the coarse stage's u_near and step as
    floats (inv_float) or per item over distinct ranges (inv_batch, inv_wide), or a per-pixel
    first rung (inv_map, inv_behind) from a smooth depth field spanning the range geometrically,
    rule 4's far clamp applied.  Ladders over the DTU range with 8, 32 or 48 planes take
    ops.inverse_steps's steps for (8, 32, 48) planes; the others sweep their range in D planes."""
    near, far = _INV_RANGE[{"inv_wide": "wide", "inv_behind": "behind"}.get(kind, "dtu")]
    nb = [near * (1 + 0.06 * b) for b in range(B)]
    fb = [far * (1 + 0.1 * b) for b in range(B)]
    dtu = kind in ("inv_float", "inv_batch") or (kind == "inv_map" and D in (8, 32, 48))
    Ds, ratios = ((8, 32, 48), (1, 2, 4)) if dtu else ((D, D, D), (1, 1, 1))
    per = kind != "inv_float"
    dmin = torch.tensor(nb[:B] if per else nb[:1]).view(-1, 1)
    dint = torch.tensor([(f - n) / ((Ds[2] - 1) * ratios[2]) for n, f in zip(nb, fb)][:B if per else 1]).view(-1, 1)
    st = ops.inverse_steps(dmin if per else float(dmin), dint if per else float(dint), Ds, ratios,
                           B, DEV)
    if kind in ("inv_float", "inv_batch", "inv_wide"):      # floats or (B,) tensors
        return ops.Ladder(st.u_near, st.step[level], D, B, h, w, DEV, inverse=True)
    ys = torch.arange(h, device=DEV, dtype=torch.float32).view(1, h, 1)
    xs = torch.arange(w, device=DEV, dtype=torch.float32).view(1, 1, w)
    bb = torch.arange(B, device=DEV, dtype=torch.float32).view(B, 1, 1)
    t = 0.5 + 0.5 * torch.sin(xs / 23.0 + bb) * torch.cos(ys / 17.0)
    t = (t + 0.05 * torch.rand(B, h, w, generator=g, device=DEV)).clamp(0, 1)
    nt, ft = torch.tensor(nb, device=DEV).view(B, 1, 1), torch.tensor(fb, device=DEV).view(B, 1, 1)
    depth = nt * (ft / nt) ** t
    s = st.step[level].view(B, 1, 1)
    first = torch.maximum(1 / depth + D / 2 * s, st.u_far.view(B, 1, 1) + (D - 1) * s)
    return ops.Ladder(first.contiguous(), st.step[level], D, B, h, w, DEV, inverse=True)


def _hyp(g, kind, B, D, h, w, step, level=0):
    """-> ops.Ladder, or a (B, D, h, w) tensor for the public warp_cost."""
    if kind.startswith("inv_"):
        return _inv_ladder(g, kind, B, D, h, w, level)
    if kind == "float":
        return ops.Ladder(425.0, step, D, B, h, w, DEV)
    if kind == "batch":
        fb = torch.tensor([425.0 + 13.7 * b for b in range(B)], device=DEV)
        sb = torch.tensor([step * (1 + 0.1 * b) for b in range(B)], device=DEV)
        return ops.Ladder(fb, sb, D, B, h, w, DEV)
    if kind == "unit":                                        # 1, 2, 3, ...: the grid pose
        return ops.Ladder(1.0, 1.0, D, B, h, w, DEV)
    if kind in ("map", "clamped", "disc"):
        return ops.Ladder(_first_map(g, B, h, w, D, step, kind), step, D, B, h, w, DEV)
    if kind == "wide":
        return ops.Ladder(_first_map(g, B, h, w, D, 12 * step, "map"), 12 * step, D, B, h, w, DEV)
    if kind == "pow2":                                       # 1, 2, 4, 1, ... per plane
        d = torch.tensor([float(2 ** (i % 3)) for i in range(D)], device=DEV)
        return d.view(1, D, 1, 1).expand(B, D, h, w).contiguous()
    if kind == "nonmono":                                    # a per-pixel shuffle of the planes
        lad = _hyp(g, "map", B, D, h, w, step).materialize()
        perm = torch.argsort(torch.rand(B, D, h, w, generator=g, device=DEV), dim=1)
        return torch.gather(lad, 1, perm).contiguous()
    raise ValueError(kind)


def _hyp_tensor(hyp):
    if not isinstance(hyp, ops.Ladder):
        return hyp
    m = hyp.materialize()
    if not hyp.inverse:
        return m
    want = torch.from_numpy(INV.ladder_f32(hyp.first, hyp.step, hyp.D, hyp.B, hyp.h, hyp.w)).to(DEV)
    assert torch.equal(m, want), "inverse Ladder.materialize() != INV.ladder_f32"
    return want


# ------------------------------------------------------------------------------- case table
# name: (entry, B, V, C, G, h, w, D, pose, hyp, family)
#   entry: ladder (warp_cost_ladder, channels-last and blocked), warp_nhwc / warp_nchw
#   (ops.warp_cost, output layout; *_nchwf: NCHW features through the transpose), homo
CASES = {}


def _add(name, *spec):
    CASES[name] = spec


_LEVELS = {0: (8, 8), 1: (16, 32), 2: (32, 48)}             # level: C, D at 640x512
_STEP = {2: 4 * synth.DEPTH_INTERVAL, 1: 2 * synth.DEPTH_INTERVAL, 0: synth.DEPTH_INTERVAL}
for _G, _cfg in ((1, "cfg2"), (8, "cfg3")):
    for _l, (_C, _D) in _LEVELS.items():
        _add(f"{_cfg}_L{_l}", "ladder", 2, 3, _C, _G, 512 >> _l, 640 >> _l, _D, "default",
             "float" if _l == 2 else "map", "staged")
    _add(f"{_cfg}_L2_batch", "ladder", 2, 3, 32, _G, 128, 160, 48, "default", "batch", "staged")
    _add(f"{_cfg}_L1_stress", "ladder", 2, 3, 16, _G, 256, 320, 32, "stress", "map", "staged")
    _add(f"{_cfg}_L0_clamped", "ladder", 2, 3, 8, _G, 512, 640, 8, "default", "clamped", "staged")
    for _l, (_C, _D) in _LEVELS.items():
        _add(f"{_cfg}_L{_l}_inv", "ladder", 2, 3, _C, _G, 512 >> _l, 640 >> _l, _D, "default",
             "inv_float" if _l == 2 else "inv_map", "staged")
    _add(f"{_cfg}_L2_inv_batch", "ladder", 2, 3, 32, _G, 128, 160, 48, "default", "inv_batch",
         "staged")
for _cfg, (_W, _H, _V, _Ds) in {"cfg4": (1152, 864, 5, (8, 32, 48)),
                                "cfg5": (1920, 1056, 7, (8, 32, 64))}.items():
    for _l in (2, 1, 0):
        _add(f"{_cfg}_L{_l}", "warp_nhwc", 2, _V, 8 << _l, 1, _H >> _l, _W >> _l, _Ds[_l],
             "default", "float" if _l == 2 else "map", "gather")
# staged kernels at 1 and 2 source views, every C, at the staging geometries
_GEOS = [("default", "map", 13, 37, 7), ("stress", "map", 22, 45, 9), ("default", "wide", 19, 70, 13),
         ("default", "disc", 24, 66, 6), ("grid", "unit", 9, 35, 4), ("default", "clamped", 12, 40, 1),
         ("stress", "float", 2, 41, 5), ("default", "batch", 17, 2, 3)]
for _V in (2, 3):
    for _C in (8, 16, 32):
        for _G in (1, 8):
            for _i, (_pose, _hk, _h, _w, _D) in enumerate(_GEOS):
                if (_i + _C // 8 + _G) % 3 and _hk not in ("wide", "disc"):
                    continue                                  # a third of the small geometries
                _add(f"staged_v{_V}_c{_C}_g{_G}_{_pose}_{_hk}", "ladder", 2, _V, _C, _G, _h, _w, _D,
                     _pose, _hk, "staged")
        _add(f"staged_v{_V}_c{_C}_nonmono", "warp_nhwc", 2, _V, _C, 1, 21, 47, 9, "default",
             "nonmono", "staged")
# the same kernels in the inverse mode: every (V, C, G) at inverse-wide, inverse-behind and one of
# the other inverse forms
_INV_GEOS = [("default", "inv_map", 13, 37, 7), ("default", "inv_float", 17, 33, 5),
             ("stress", "inv_batch", 9, 40, 9)]
for _V in (2, 3):
    for _C in (8, 16, 32):
        for _G in (1, 8):
            _add(f"staged_v{_V}_c{_C}_g{_G}_inv_wide", "ladder", 2, _V, _C, _G, 24, 160, 3,
                 "default", "inv_wide", "staged")
            _add(f"staged_v{_V}_c{_C}_g{_G}_inv_behind", "ladder", 2, _V, _C, _G, 16, 96, 9,
                 "stress", "inv_behind", "staged")
            _pose, _hk, _h, _w, _D = _INV_GEOS[(_V + _C // 8 + _G) % 3]
            _add(f"staged_v{_V}_c{_C}_g{_G}_{_pose}_{_hk}", "ladder", 2, _V, _C, _G, _h, _w, _D,
                 _pose, _hk, "staged")
# gather kernels: 1, 2, 4, 6 source views x C x variance / group-wise x output layout;
# group sizes C/G in {1, 2, 4, 8, 16, 32} over the table
_GW = {("nchw", 8): 8, ("nhwc", 8): 2, ("nchw", 16): 8, ("nhwc", 16): 2, ("nchw", 32): 8,
       ("nhwc", 32): 2, ("nchw", 64): 2, ("nhwc", 64): 4}
_SHAPES = [(13, 37, 7, "default", "map"), (2, 29, 5, "stress", "map"), (17, 2, 3, "grid", "pow2"),
           (9, 33, 1, "default", "float"), (21, 19, 13, "stress", "nonmono"),
           (11, 26, 6, "grid", "pow2")]
_k = 0
for _ns in (1, 2, 4, 6):
    for _C in (8, 16, 32, 64):
        for _out in ("nchw", "nhwc"):
            for _G in (1, _GW[(_out, _C)]):
                if _out == "nhwc" and _G == 1 and _ns <= 2 and _C <= 32:
                    continue                                  # the staged kernel: the child below
                _h, _w, _D, _pose, _hk = _SHAPES[_k % len(_SHAPES)]
                _k += 1
                _add(f"gather_s{_ns}_c{_C}_g{_G}_{_out}", f"warp_{_out}", 2, _ns + 1, _C, _G, _h, _w,
                     _D, _pose, _hk, "gather")
for _ns in (3, 5, 15):
    for _out in ("nchw", "nhwc"):
        for _G in (1, 4):
            _add(f"generic_s{_ns}_g{_G}_{_out}", f"warp_{_out}" + ("_nchwf" if _G == 4 else ""), 2,
                 _ns + 1, 16, _G, 10, 23, 5, "stress" if _out == "nchw" else "default", "map",
                 "gather")
for _C, _pose, _hk in ((8, "grid", "pow2"), (16, "stress", "map"), (32, "default", "nonmono")):
    _add(f"homo_c{_C}_{_pose}", "homo", 2, 2, _C, 1, 14, 31, 6, _pose, _hk, "homo")

# gather-kernel variance at 1 or 2 source views with NHWC output: CASMVS_K1_SMEM=0 only
CHILD = {f"gather_smem0_s{_ns}_c{_C}": ("warp_nhwc", 2, _ns + 1, _C, 1, 15, 34, 7, _pose, "map",
                                         "gather")
         for _ns in (1, 2) for _C, _pose in ((8, "default"), (16, "stress"), (32, "default"))}


def _inputs(name, spec):
    entry, B, V, C, G, h, w, D, pose, hk, fam = spec
    g = torch.Generator(device=DEV).manual_seed(_seed(name))
    level = {8: 0, 16: 1, 32: 2}.get(C, 1)
    W_, H = w << level, h << level
    feats = _feats(g, B, V, C, h, w, nchw=entry.endswith("_nchwf"))
    P = _proj(pose, V, W_, H, level, B)
    hyp = _hyp(g, hk, B, D, h, w, _STEP[level], level)
    if entry != "ladder" and isinstance(hyp, ops.Ladder):
        hyp = hyp.materialize()
    return feats, P, hyp


# The staged kernels' pixel tile (TW, TH) per C and their box: BW = TW + 16 columns, rounded up to
# a 1024-byte row for the plane-group kernel (2 source views, variance), BH = TH + 4 rows
# (warp_cost_smem.cu: kShapes and launch()).
_TILE = {8: (32, 4), 16: (32, 2), 32: (16, 2)}


def _box(V, C, G):
    tw, th = _TILE[C]
    wq = 1024 // (C * 4) if (V == 3 and G == 1) else 1
    return tw, th, -(-(tw + 16) // wq) * wq, th + 4


def _samples(P, dv):
    """Float64 source coordinates of every (b, view, plane, y, x) as the kernels form them:
    q = R (x, y, 1) + t / d, u = q_x / q_z -> (u, v, q_z)."""
    P, dv = P.double().cpu(), dv.double().cpu()
    B, D, h, w = dv.shape
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64),
                            indexing="ij")
    pix = torch.stack([xs, ys, torch.ones_like(xs)], 0).view(3, -1)                 # (3, hw)
    a = (P[..., :3] @ pix).view(B, -1, 3, 1, h, w)                                    # (B,S,3,1,h,w)
    q = a + P[..., 3].view(B, -1, 3, 1, 1, 1) / dv.view(B, 1, 1, D, h, w)
    return q[:, :, 0] / q[:, :, 2], q[:, :, 1] / q[:, :, 2], q[:, :, 2]


def _wide(spec, P, dv):
    """Planes 0 and 1 alone already need more than the staged box in some tile and view: the
    kernel's first run, whatever its length, is halved down to single planes."""
    _, B, V, C, G, h, w = spec[:7]
    tw, th, bw, bh = _box(V, C, G)
    u, v, qz = (t[:, :, :2] for t in _samples(P, dv))
    ok = (qz > 1e-7) & (u > -2) & (u < w + 1) & (v > -2) & (v < h + 1)
    hp, wp = -(-h // th) * th, -(-w // tw) * tw
    spans = []
    for t in (u.floor(), v.floor()):
        big = torch.where(ok, t, torch.full_like(t, float("nan")))
        big = torch.nn.functional.pad(big, (0, wp - w, 0, hp - h), value=float("nan"))
        tiles = big.reshape(*big.shape[:3], hp // th, th, wp // tw, tw).transpose(4, 5)
        tiles = tiles.reshape(*tiles.shape[:5], -1).flatten(2, 2)
        tiles = tiles.permute(0, 1, 3, 4, 2, 5).flatten(4)                  # (B,S,ty,tx,2*th*tw)
        mx = torch.where(tiles.isnan(), -torch.inf, tiles).amax(-1)
        mn = torch.where(tiles.isnan(), torch.inf, tiles).amin(-1)
        spans.append(mx + 2 - mn)
    return bool(((spans[0] > bw) | (spans[1] > bh)).any())


def _behind(spec, P, dv):
    """Part of the sweep lies behind a source camera (q_z <= 1e-7), part in front of it."""
    qz = _samples(P, dv)[2]
    return bool((qz <= 1e-7).any()) and bool((qz > 1e-7).any())


INV_EDGES = {"inv_wide": _wide, "inv_behind": _behind}


def _cl5(feats):
    """logical (B, V, C, h, w) -> (B, V, h, w, C) values."""
    return feats.permute(0, 1, 3, 4, 2)


def _launch(spec, feats, P, hyp):
    """Runs the case's kernels: {label: (unrounded, rounded or None)} as (B, D, h, w, Cout)."""
    entry, B, V, C, G, h, w, D = spec[:8]
    out = {}
    if entry == "ladder":
        for blocked in (False, True):
            y = [ops.warp_cost_ladder(feats, P, hyp, G, round_tf32=r, blocked=blocked) for r in (False, True)]
            y = [W.from_blocked(t) if blocked else ops.volume_storage(t) for t in y]
            out["blocked" if blocked else "cl"] = tuple(y)
    elif entry.startswith("warp"):
        lay = ops.NCHW if entry.startswith("warp_nchw") else ops.NHWC
        y = [ops.warp_cost(feats, P, hyp, G, lay, round_tf32=r) for r in (False, True)]
        out[entry] = tuple(ops.volume_storage(t) for t in y)
    elif entry == "homo":
        src = feats[:, 1]
        P0 = P[:, 0].contiguous()
        y_nchw = ops.homo_warp(src.contiguous(), P0, hyp)                    # transpose + NCHW out
        y_nhwc = torch.empty(B, D, h, w, C, device=DEV)
        src_cl = src.permute(0, 2, 3, 1).contiguous()
        _lib.check(_lib.load().casmvs_homo_warp_fwd(ops._ptr(src_cl), ops.NHWC, ops._ptr(P0),
                                                    ops._ptr(hyp), ops._ptr(y_nhwc), ops.NHWC, B, C,
                                                    D, h, w, ops._stream()), "homo_warp")
        out["nchw"] = (y_nchw.permute(0, 2, 3, 4, 1), None)
        out["nhwc"] = (y_nhwc, None)
    return out


def _check_outputs(name, spec, feats, P, hyp, out):
    entry, B, V, C, G = spec[:5]
    fam = spec[-1]
    f = _cl5(feats)
    dv = _hyp_tensor(hyp)
    reps = []
    first = None
    for label, (y, yr) in out.items():
        if yr is not None:
            want = W.tf32_rna(y.contiguous())
            assert torch.equal(yr.contiguous().view(torch.int32), want.view(torch.int32)), \
                f"{name}/{label}: TF32-rounded store differs from tf32_rna of the unrounded output"
        if first is not None and entry in ("ladder", "homo"):
            # blocked vs channels-last, NCHW vs NHWC: the same arithmetic, bit for bit
            assert torch.equal(y, first), f"{name}/{label}: differs from the other layout"
            continue
        first = y
        if entry == "homo":
            rep = W.check_homo_warp(y, f[:, 1], P[:, 0], dv, EPS[fam])
        else:
            rep = W.check_cost(y, f, P, dv, G, EPS[fam])
        print(f"[k1-fp64] {name}/{label} [{fam}]: {rep.describe()}")
        reps.append(rep)
    return reps


def _assert(name, spec, reps):
    fam = spec[-1]
    for rep in reps:
        assert rep.ok, f"{name} [{fam}]: {rep.describe()}"
        assert rep.loose_share <= LOOSE_CEIL["cost"], f"{name} [{fam}] loose: {rep.describe()}"


@pytest.mark.parametrize("name", list(CASES))
def test_k1_vs_fp64(name):
    spec = CASES[name]
    feats, P, hyp = _inputs(name, spec)
    hk = spec[9]
    if hk in INV_EDGES:
        dv = _hyp_tensor(hyp).cpu()
        assert INV_EDGES[hk](spec, P, dv), f"{name}: {hk} does not hold"
    out = _launch(spec, feats, P, hyp)
    _assert(name, spec, _check_outputs(name, spec, feats, P, hyp, out))


# ------------------------------------------------------------------------------- child process
def _child_main(path):
    """CASMVS_K1_SMEM=0: the CHILD cases, their outputs and the kernels launched."""
    from torch.profiler import ProfilerActivity, profile
    res = {}
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, spec in CHILD.items():
            feats, P, hyp = _inputs(name, spec)
            res[name] = {k: tuple(t.cpu() if t is not None else None for t in v)
                         for k, v in _launch(spec, feats, P, hyp).items()}
        torch.cuda.synchronize()
    names = sorted({e.name for e in prof.events()})
    torch.save({"out": res, "kernels": names}, path)


@pytest.fixture(scope="module")
def child(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("k1") / "child.pt")
    code = ("import sys\nsys.path.insert(0, %r)\nsys.path.insert(0, %r)\n"
            "import test_gpu_warp_cost_fp64 as T\nT._child_main(sys.argv[1])\n"
            % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, CASMVS_K1_SMEM="0")
    subprocess.run([sys.executable, "-c", code, path], check=True, env=env, timeout=600)
    return torch.load(path)


@pytest.mark.parametrize("name", list(CHILD))
def test_gather_variance_nhwc_small_views_vs_fp64(child, name):
    spec = CHILD[name]
    feats, P, hyp = _inputs(name, spec)
    out = {k: tuple(t.to(DEV) if t is not None else None for t in v) for k, v in child["out"][name].items()}
    _assert(name, spec, _check_outputs(name, spec, feats, P, hyp, out))


# ------------------------------------------------------------------------------- coverage
def _expected_kernels():
    exp = set()
    for c in (8, 16, 32):
        for blk in (False, True):
            for inv in (False, True):
                exp.add(("smem", 1, c, False, blk, inv))
                exp.add(("smem", 1, c, True, blk, inv))
                exp.add(("smem", 2, c, True, blk, inv))
                exp.add(("smem_pg", 2, c, False, blk, inv))
    for ns in (1, 2, 4, 6):
        for ct in (8, 16, 32, 0):
            for gwc in (False, True):
                for nhwc in (False, True):
                    exp.add(("gather", ns, ct, gwc, nhwc))
    for gwc in (False, True):
        for nhwc in (False, True):
            exp.add(("gather", 0, 0, gwc, nhwc))
    exp |= {("homo", False), ("homo", True), ("transpose",), ("bwd", False), ("bwd", True)}
    return exp


def _parse_kernels(names):
    b = lambda s: s == "true"                                           # noqa: E731
    got = set()
    for n in names:
        m = re.search(r"warp_var_smem(_inv)?_kernel<(\d+), (\d+), \d+, \d+, \d+, (true|false), "
                      r"(true|false)>", n)
        if m:
            got.add(("smem", int(m[2]), int(m[3]), b(m[4]), b(m[5]), bool(m[1])))
        m = re.search(r"warp_var_smem_pg(_inv)?_kernel<(\d+), \d+, \d+, \d+, \d+, (true|false)>", n)
        if m:
            got.add(("smem_pg", 2, int(m[2]), False, b(m[3]), bool(m[1])))
        m = re.search(r"warp_cost_kernel<(\d+), (\d+), (true|false), (true|false)>", n)
        if m:
            got.add(("gather", int(m[1]), int(m[2]), b(m[3]), b(m[4])))
        m = re.search(r"homo_warp_kernel<(true|false)>", n)
        if m:
            got.add(("homo", b(m[1])))
        m = re.search(r"warp_cost_bwd_kernel<(true|false)>", n)
        if m:
            got.add(("bwd", b(m[1])))
        if "transpose_rs_kernel" in n:
            got.add(("transpose",))
    return got


def test_every_k1_instantiation_launched(child):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, spec in CASES.items():
            _launch(spec, *_inputs(name, spec))
        for name, spec in BWD.items():
            _bwd_launch(spec, *_bwd_inputs(name, spec))
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()} | set(child["kernels"])
    got = _parse_kernels(names)
    missing = sorted(_expected_kernels() - got, key=str)
    staged = {k for k in _expected_kernels() if k[0].startswith("smem")}
    print(f"[k1-fp64] {len(got & _expected_kernels())} of {len(_expected_kernels())} K1 "
          f"instantiations launched, {len(got & staged)} of {len(staged)} staged (uniform and "
          f"inverse)")
    assert not missing, f"never launched: {missing}"


# ------------------------------------------------------------------------------- backward
# name: (B, V, C, G, h, w, D, pose)
BWD = {}
for _l, (_C, _D) in _LEVELS.items():
    for _G in (1, 8):
        for _B, _pose in ((1, "default"), (2, "default"), (2, "stress")):
            BWD[f"train_L{_l}_g{_G}_b{_B}_{_pose}"] = (_B, 3, _C, _G, 512 >> _l, 640 >> _l, _D, _pose)
for _ns in (4, 15):
    for _G in (1, 8):
        BWD[f"small_s{_ns}_g{_G}"] = (2, _ns + 1, 16, _G, 11, 27, 5, "stress")


def _bwd_inputs(name, spec):
    B, V, C, G, h, w, D, pose = spec
    g = torch.Generator(device=DEV).manual_seed(_seed(name))
    level = {8: 0, 16: 1, 32: 2}[C]
    f = torch.randn(B, V, h, w, C, generator=g, device=DEV)
    P = _proj(pose, V, w << level, h << level, level, B)
    dv = _hyp(g, "map", B, D, h, w, _STEP[level]).materialize()
    gcost = torch.randn(B, D, h, w, C if G == 1 else G, generator=g, device=DEV)
    return f, P, dv, gcost


def _bwd_launch(spec, f, P, dv, gcost):
    B, V, C, G, h, w, D, _ = spec
    gf = torch.zeros_like(f)
    _lib.check(_lib.load().casmvs_warp_cost_bwd(ops._ptr(f), ops._ptr(P), ops._ptr(dv), ops._ptr(gcost),
                                                ops._ptr(gf), B, V, C, D, h, w, G, ops._stream()),
               "warp_cost_bwd")
    return gf


@pytest.mark.parametrize("name", list(BWD))
def test_warp_cost_bwd_vs_fp64(name):
    spec = BWD[name]
    f, P, dv, gcost = _bwd_inputs(name, spec)
    gf = _bwd_launch(spec, f, P, dv, gcost)
    rep = W.check_warp_cost_bwd(gf, f, P, dv, gcost, spec[3], EPS["bwd"])
    print(f"[k1-fp64] {name} [bwd]: {rep.describe()}")
    assert rep.ok, f"{name}: {rep.describe()}"
    assert rep.loose_share <= LOOSE_CEIL["bwd"], f"{name} loose: {rep.describe()}"
