"""The two training losses element by element against float64 at the shapes, view counts, top-K
values and level counts they accept, not only at the ones training uses by default.

Photometric loss (csrc/photo_loss.cu).  Each case of PHOTO_CASES names the edges it exists for;
test_photo_case_table_edges asserts every one of them by construction on the CPU: tiles cut by
the right or bottom edge, odd level sizes, a 3x3 level, 1, 2 and 4 levels, one and sixteen
source views (the selection mask's top bit), K = S > 4, a batch of three with a distinct depth
interval per sample, two sources whose e is bit-equal, a source seen through the reference's
own camera (samples on the clamped tap), a source behind which part of the image warps,
NaN, +inf, zero and negative depths (and +inf without NaN, so S_l is +inf at some levels and
finite at another), one level without a valid pixel, and smoothness weights 0 and 10.  Every
case runs losses.photo_loss with its debug maps and goes through
test_gpu_photo_loss.check_against_fp64, at that file's tolerances.  Then one seeded train.main
step of --loss_type photo on a textured COLMAP capture at 800x608, checked with the same helper
on the recorded call's own inputs, and the capture's projections against the COLMAP cameras.

SL1 loss and depth metrics (csrc/loss.cu) at 640x512 (B = 1, 2, 4), 768x576 (B = 4) and
1600x1184 (B = 1), so the grid-stride loop runs many passes, at 1, 2, 3 and 4 levels, with
random, all-true and empty masks and differences placed exactly at +-0.5, 1, 2 and 4: the loss
within one float32 spacing of float64, the counts exact with strict <, the |e| sum equal to
float32 of the exact sum, the gradient bit for bit equal to a float32 restatement of ATen's
smooth_l1_backward (checked on the CPU against torch) and within its three float32 roundings
(3 * 2^-24 relative) of the float64 derivative, and depth_metrics equal to level 0's metrics."""
import inspect
import math

import cv2
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_gpu_photo_loss as PL
from casmvsnet_pl_b200 import io, losses, synth, synth_scenes, train, train_data
from oracle import photo_loss_fp64 as O
from test_gpu_photo_loss import GRAD_ABS, GRAD_REL, OVER_SHARE_MAX, VALID_MISMATCH_MAX  # noqa: F401

DEV = "cuda:0"
TILE = 16                      # kPhotoTile
MAX_SOURCES = 16               # kPhotoMaxSources: bit 15 of the uint16 selection mask


@pytest.fixture(autouse=True)
def _grad_mode():
    with torch.enable_grad():            # conftest runs GPU tests under no_grad by default
        yield


# ------------------------------------------------------------------------------- case table
# name: image W, H, levels, views V, top-K, batch B, and optionally: step (degrees between the
# arc cameras; synth's DTU layout when absent), identity (sources seen through the reference's
# own camera, P = [I | 0]), twin (source b a bit-exact copy of source a: image and projection),
# behind_view (synth.projection_matrices), amp (depth amplitude around the convergence depth),
# nonfinite, empty_level, lam, ratios; edges lists what the case exists for (EDGES)
PHOTO_CASES = {
    "cli_small": dict(W=160, H=128, levels=3, V=3, K=1, B=1, edges=("x_partial",)),
    "cli_800": dict(W=800, H=608, levels=3, V=4, K=2, B=3,
                    edges=("x_partial", "y_partial", "batch3", "distinct_dint")),
    "full_dtu": dict(W=1600, H=1184, levels=3, V=2, K=1, B=1, edges=("S1", "y_partial")),
    "odd": dict(W=100, H=76, levels=3, V=3, K=2, B=2, ratios=(1.0, 2.5, 5.5),
                edges=("odd_dims", "partial_every_level")),
    "tiny": dict(W=12, H=12, levels=3, V=3, K=1, B=2, identity=(1,), edges=("level_3x3",)),
    "four_levels": dict(W=72, H=24, levels=4, V=3, K=1, B=1, identity=(1,),
                        edges=("levels4", "level_9x3")),
    "one_level": dict(W=64, H=48, levels=1, V=3, K=2, B=2, edges=("levels1",)),
    "two_levels": dict(W=64, H=48, levels=2, V=3, K=2, B=2, edges=("levels2",)),
    "many_sources_k16": dict(W=256, H=192, levels=3, V=17, K=16, B=1, step=0.5,
                             edges=("S16", "K_eq_S", "K_gt4")),
    "many_sources_k9": dict(W=256, H=192, levels=3, V=17, K=9, B=1, step=0.5, edges=("S16", "K_gt4")),
    "ties_and_taps": dict(W=160, H=128, levels=3, V=4, K=1, B=2, step=2.0, twin=(0, 1), identity=(2,),
                          edges=("ties", "clamped_tap")),
    "behind": dict(W=320, H=256, levels=3, V=3, K=1, B=1, behind_view=1, amp=120.0, edges=("behind",)),
    "nonfinite": dict(W=96, H=80, levels=3, V=3, K=2, B=2, nonfinite="all", edges=("nonfinite",)),
    "nonfinite_inf": dict(W=96, H=80, levels=3, V=3, K=2, B=2, nonfinite="inf", edges=("inf_without_nan",)),
    "one_level_empty": dict(W=160, H=128, levels=3, V=3, K=1, B=2, empty_level=1,
                            edges=("one_level_empty",)),
    "lambda0": dict(W=160, H=128, levels=3, V=3, K=2, B=2, lam=0.0, edges=("lambda0",)),
    "lambda10": dict(W=160, H=128, levels=3, V=3, K=2, B=2, lam=10.0, edges=("lambda10",)),
}
DINT = (2.65, 3.1, 1.9, 2.2)


def dims(c):
    """[(w_l, h_l)] of every level."""
    return [(c["W"] >> l, c["H"] >> l) for l in range(c["levels"])]


def photo_cameras(c):
    """(S, levels, 3, 4) float32: synth's DTU layout (or its arc at c['step'] degrees), with the
    identity sources replaced by [I | 0] and source twin[1] a copy of source twin[0]."""
    V, W, H, levels = c["V"], c["W"], c["H"], c["levels"]
    if "step" not in c:
        pm = synth.projection_matrices(V, W, H, levels, behind_view=c.get("behind_view")).numpy()
    else:
        pm = np.zeros((V - 1, levels, 3, 4), np.float32)
        for i in range(1, V):
            theta = math.radians((-1) ** i * c["step"] * math.ceil(i / 2))
            R = synth._rot_y(theta)
            t = np.array([-synth.CONVERGE_MM * math.sin(theta), 0.0, synth.CONVERGE_MM * (1 - math.cos(theta))])
            for l in range(levels):
                K = synth.intrinsics(l, W, H)
                src, ref = np.eye(4), np.eye(4)
                src[:3, :4] = K @ np.concatenate([R, t[:, None]], 1)
                ref[:3, :3] = K
                pm[i - 1, l] = (src @ np.linalg.inv(ref))[:3, :4]
    for s in c.get("identity", ()):
        pm[s] = np.eye(3, 4, dtype=np.float32)
    if "twin" in c:
        a, b = c["twin"]
        pm[b] = pm[a]
    return torch.from_numpy(np.ascontiguousarray(pm))


NONFINITE = {   # kind -> the values placed at each level
    "all": lambda l: [float("nan"), float("inf"), 0.0, -5.0],
    # no NaN: +inf at levels 0 and 1 (S_l = +inf there), level 2 non-positive only (S_2 finite)
    "inf": lambda l: [float("inf"), 0.0, -5.0] if l < 2 else [0.0, -5.0],
}


def nonfinite_spots(w, h, vals):
    """(x, y, value) of the non-finite and non-positive depths at a level, `vals` in turn:
    interior pixels, the border, and both sides of the tile seam x = 16 (y = 16); no two
    spots are neighbours."""
    spots = [(w // 2, h // 2), (w // 3, h // 2 + 1), (0, h // 2), (w - 1, 1), (w // 2, 0), (3, h - 1)]
    if w > TILE + 1:
        spots += [(TILE - 1, h // 3), (TILE, h // 3 + 2)]
    if h > TILE + 1:
        spots += [(w // 4, TILE - 1), (w // 4 + 2, TILE)]
    return [(x, y, vals[i % len(vals)]) for i, (x, y) in enumerate(spots)]


def photo_inputs(c, device=DEV, seed=0):
    """imgs (B,V,3,H,W) normalised blurred noise, proj_mats (B,S,levels,3,4), depths per level
    (smooth around the convergence depth, different per level and sample, with the case's
    non-finite spots or empty level), dint (B,1) distinct per sample."""
    B, V, W, H = c["B"], c["V"], c["W"], c["H"]
    rng = np.random.default_rng(seed)
    u8 = np.stack([cv2.GaussianBlur(rng.integers(0, 256, (H, W, 3), dtype=np.uint8), (0, 0), 2.0)
                   for _ in range(B * V)]).reshape(B, V, H, W, 3)
    if "twin" in c:
        a, b = c["twin"]
        u8[:, b + 1] = u8[:, a + 1]
    u8 = torch.from_numpy(u8.reshape(B * V, H, W, 3))
    if device == "cpu":          # the CPU edge checks: the arithmetic io.normalize_images matches
        mean, std = (torch.tensor(t).view(3, 1, 1) for t in (io.IMAGENET_MEAN, io.IMAGENET_STD))
        imgs = u8.permute(0, 3, 1, 2).float().div(255).sub(mean).div(std).view(B, V, 3, H, W)
    else:
        imgs = io.normalize_images(u8.to(device)).view(B, V, 3, H, W)
    pm = photo_cameras(c).unsqueeze(0).expand(B, -1, -1, -1, -1).contiguous().to(device)
    amp = c.get("amp", 40.0)
    depths = []
    for l, (w, h) in enumerate(dims(c)):
        ys, xs = np.mgrid[0:h, 0:w].astype(np.float64) * (1 << l)
        d = np.stack([synth.CONVERGE_MM + amp * np.sin(xs / 37 + b) * np.cos(ys / 53) + 3 * l
                      + rng.normal(0, 0.5, xs.shape) for b in range(B)]).astype(np.float32)
        if c.get("nonfinite"):
            for b in range(B):
                for x, y, val in nonfinite_spots(w, h, NONFINITE[c["nonfinite"]](l)):
                    d[b, y, x] = val
        if c.get("empty_level") == l:
            d = -d
        depths.append(torch.from_numpy(d).to(device))
    dint = torch.tensor([[v] for v in DINT[:B]], device=device)
    return imgs, pm, depths, dint


def _pz(pm, d, l):
    """p_z (B,S,h,w) float64 of every pixel of level l with depth d (B,h,w)."""
    P = pm[:, :, l].double()
    B, S = P.shape[:2]
    h, w = d.shape[1:]
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64),
                            indexing="ij")
    m = P[:, :, 2, :, None, None]
    return m[:, :, 0] * xs + m[:, :, 1] * ys + m[:, :, 2] + m[:, :, 3] / d.double()[:, None]


EDGES = {
    "x_partial": lambda c, _: any(w % TILE for w, _ in dims(c)),
    "y_partial": lambda c, _: any(h % TILE for _, h in dims(c)),
    "partial_every_level": lambda c, _: all(w % TILE and h % TILE for w, h in dims(c)),
    "odd_dims": lambda c, _: any(w % 2 and h % 2 for w, h in dims(c)),
    "level_3x3": lambda c, _: (3, 3) in dims(c),
    "level_9x3": lambda c, _: (9, 3) in dims(c),
    "levels1": lambda c, _: c["levels"] == 1,
    "levels2": lambda c, _: c["levels"] == 2,
    "levels4": lambda c, _: c["levels"] == 4,
    "S1": lambda c, _: c["V"] - 1 == 1,
    "S16": lambda c, _: c["V"] - 1 == MAX_SOURCES,
    "K_eq_S": lambda c, _: c["K"] == c["V"] - 1,
    "K_gt4": lambda c, _: c["K"] > 4,
    "batch3": lambda c, _: c["B"] == 3,
    "distinct_dint": lambda c, inp: c["B"] > 1 and len(set(inp[3].flatten().tolist())) == c["B"],
    # sources a and b see bit-identical images through bit-identical projections
    "ties": lambda c, inp: (torch.equal(inp[0][:, c["twin"][0] + 1], inp[0][:, c["twin"][1] + 1])
                            and torch.equal(inp[1][:, c["twin"][0]], inp[1][:, c["twin"][1]])),
    # u = x and v = y exactly, valid up to the last column and row, so they sample x1 = w - 1
    "clamped_tap": lambda c, inp: all(_identity_warp(inp, s, l) for s in c["identity"]
                                      for l in range(c["levels"])),
    "behind": lambda c, inp: all(bool((_pz(inp[1], d, l)[:, c["behind_view"] - 1] <= 1e-7).any())
                                 and bool((_pz(inp[1], d, l)[:, c["behind_view"] - 1] > 1e-7).any())
                                 for l, d in enumerate(inp[2])),
    "nonfinite": lambda c, inp: all(_nonfinite_placed(d, TILE) for d in inp[2]),
    # +inf depths (S_l = +inf) with no NaN anywhere, and a level whose S_l stays finite
    "inf_without_nan": lambda c, inp: (not any(torch.isnan(d).any() for d in inp[2])
                                       and bool(torch.isposinf(inp[2][0]).any())
                                       and any(bool(torch.isfinite(d).all()) for d in inp[2])
                                       and all(bool((d <= 0).any()) for d in inp[2])),
    "one_level_empty": lambda c, inp: all(bool((d <= 0).all()) == (l == c["empty_level"])
                                          and bool((d > 0).any()) == (l != c["empty_level"])
                                          for l, d in enumerate(inp[2])),
    "lambda0": lambda c, _: c["lam"] == 0.0,
    "lambda10": lambda c, _: c["lam"] == 10.0,
}


def _identity_warp(inp, s, l):
    _, pm, depths, _ = inp
    d = depths[l]
    h, w = d.shape[1:]
    u, v, ok, _, _ = O.warp(d, pm[:, s:s + 1, l], w, h)
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64),
                            indexing="ij")
    return (torch.equal(u[:, 0], xs.expand_as(u[:, 0])) and torch.equal(v[:, 0], ys.expand_as(v[:, 0]))
            and bool(ok[:, 0, :, w - 1].all()) and bool(ok[:, 0, h - 1].all()))


def _nonfinite_placed(d, tile):
    """NaN, +inf, 0 and a negative depth all occur; on the border, in the interior, and (where
    the level is wider or taller than a tile) on both sides of a tile seam."""
    bad = ~(torch.isfinite(d) & (d > 0))
    h, w = d.shape[1:]
    kinds = (torch.isnan(d).any() and torch.isposinf(d).any() and (d == 0).any() and (d < 0).any())
    border = bad[:, 0].any() or bad[:, -1].any() or bad[:, :, 0].any() or bad[:, :, -1].any()
    interior = bad[:, 1:-1, 1:-1].any()
    seam = w <= tile + 1 or (bad[:, :, tile - 1].any() and bad[:, :, tile].any())
    seam_y = h <= tile + 1 or (bad[:, tile - 1].any() and bad[:, tile].any())
    return bool(kinds and border and interior and seam and seam_y)


def test_photo_case_table_edges():
    """Every edge a case names holds for the case's parameters and its inputs (built on the CPU),
    and every edge is named by some case."""
    named = set()
    for name, c in PHOTO_CASES.items():
        inp = photo_inputs(c, device="cpu")
        for e in c["edges"]:
            assert EDGES[e](c, inp), f"{name}: edge {e} does not hold"
            named.add(e)
        assert 1 <= c["K"] <= c["V"] - 1 <= MAX_SOURCES and 1 <= c["levels"] <= 4
        assert all(w >= 3 and h >= 3 for w, h in dims(c)), name
    assert named == set(EDGES)


def _valid_somewhere(c, dbg):
    """Every level except the case's empty one has valid pairs (the comparison is not vacuous)."""
    for l, k in enumerate(dbg):
        assert bool(k["valid"].any()) == (l != c.get("empty_level")), (l, int(k["valid"].sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PHOTO_CASES))
def test_photo_case_vs_fp64(name):
    c = PHOTO_CASES[name]
    imgs, pm, depths, dint = photo_inputs(c)
    ratios = c.get("ratios", (1.0, 2.0, 4.0, 8.0))[:c["levels"]]
    lam = c.get("lam", PL.LAM)
    (loss, stats, dbg), grads = PL.run(imgs, pm, depths, dint, c["K"], debug=True, ratios=ratios, lam=lam)
    _valid_somewhere(c, dbg)
    if name == "ties_and_taps":
        a, b = c["twin"]
        for k in dbg:
            assert torch.equal(k["valid"][:, a], k["valid"][:, b])
            ea, eb = k["e"][:, a], k["e"][:, b]
            assert torch.equal(ea[k["valid"][:, a]].view(torch.int32), eb[k["valid"][:, b]].view(torch.int32))
            # K = 1: of two bit-equal e the lower source index wins, so b is never selected
            assert not k["selected"][:, b].any()
            assert k["selected"][:, a].any()
        assert dbg[0]["selected"][:, c["identity"][0]].any()
    if name == "many_sources_k16":
        # the mask's top bit: source 15 is selected wherever it is valid (K = S)
        assert torch.equal(dbg[0]["selected"][:, MAX_SOURCES - 1], dbg[0]["valid"][:, MAX_SOURCES - 1])
        assert dbg[0]["valid"][:, MAX_SOURCES - 1].any()
    if name == "nonfinite":          # a NaN depth: S_l and the loss NaN, the gradient finite
        assert torch.isnan(loss) and torch.isnan(stats[:, 1]).all()
        assert all(torch.isfinite(g).all() for g in grads)
    if name == "nonfinite_inf":      # +inf depths: S_l and the loss +inf, the gradient finite
        assert loss.item() == float("inf") and stats[:2, 1].tolist() == [float("inf")] * 2
        assert torch.isfinite(stats[2]).all() and torch.isfinite(stats[:, 0]).all()
        assert all(torch.isfinite(g).all() for g in grads)
    if name == "lambda0":
        ds = [d.clone().requires_grad_(True) for d in depths]
        loss_s, stats_s = losses.photo_loss({f"depth_{l}": d for l, d in enumerate(ds)}, imgs, pm, dint, ratios,
                                            c["levels"], c["K"], 0.0)
        assert torch.equal(stats_s, stats)
    worst = PL.check_against_fp64(imgs, pm, depths, dint, ratios, c["K"], lam, loss, stats, dbg, grads, name)
    print(f"[photo {name}] largest e error / bound {max(r for r, _ in worst):.3e}, largest gradient "
          f"error / level max {max(g for _, g in worst):.3e}")


# ------------------------------------------------------------------ a real photometric training step
TRAIN_WH = (800, 608)


@pytest.fixture(scope="module")
def textured_capture(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("photo_800"))
    synth_scenes.make_colmap(root, n_views=7, image_wh=TRAIN_WH, n_points=3000, seed=11, textured=True)
    return root


@pytest.fixture
def photo_rec(monkeypatch):
    """Records the first _PhotoLossFn call: its inputs, loss, stats, incoming gradient and the
    depth gradients its backward returns."""
    calls = []
    fn = losses._PhotoLossFn
    fwd0, bwd0 = fn.forward, fn.backward

    def forward(ctx, levels, topk, smooth_weight, interval_ratios, debug_maps, imgs, proj_mats,
                depth_interval, *depths):
        out = fwd0(ctx, levels, topk, smooth_weight, interval_ratios, debug_maps, imgs, proj_mats,
                   depth_interval, *depths)
        ctx.rec = not calls and depths[0].requires_grad        # the first training step
        if ctx.rec:
            calls.append(dict(levels=levels, K=topk, lam=smooth_weight, ratios=list(interval_ratios),
                              imgs=imgs.detach().clone(), pm=proj_mats.detach().clone(),
                              dint=torch.as_tensor(depth_interval).detach().clone(),
                              depths=[d.detach().clone() for d in depths], loss=out[0].detach().clone(),
                              stats=out[1].detach().clone()))
        return out

    def backward(ctx, grad_loss, grad_stats):
        out = bwd0(ctx, grad_loss, grad_stats)
        if ctx.rec and "grads" not in calls[0]:
            calls[0]["grad_loss"] = grad_loss.detach().clone()
            calls[0]["grads"] = [g.detach().clone() for g in out[8:]]
        return out

    forward.__signature__ = inspect.signature(fwd0)
    monkeypatch.setattr(fn, "forward", staticmethod(forward))
    monkeypatch.setattr(fn, "backward", staticmethod(backward))
    return calls


@pytest.mark.gpu
def test_photo_training_step_vs_fp64(textured_capture, photo_rec, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    train.main(["--dataset_name", "colmap", "--loss_type", "photo", "--root_dir", textured_capture,
                "--img_wh", str(TRAIN_WH[0]), str(TRAIN_WH[1]), "--n_views", "5", "--photo_topk", "2",
                "--num_epochs", "1", "--log_every", "1", "--optimizer", "adam", "--exp_name", "step800", "--seed", "0"])
    call = photo_rec[0]
    assert "grads" in call and call["K"] == 2 and call["levels"] == 3
    assert tuple(call["imgs"].shape) == (1, 5, 3, TRAIN_WH[1], TRAIN_WH[0])
    # the debug maps of the same inputs: same loss, stats and gradients, bit for bit
    ds = [d.clone().requires_grad_(True) for d in call["depths"]]
    loss, stats, dbg = losses.photo_loss({f"depth_{l}": d for l, d in enumerate(ds)}, call["imgs"], call["pm"],
                                         call["dint"], call["ratios"], 3, 2, call["lam"], debug=True)
    loss.backward(call["grad_loss"])
    assert torch.equal(loss, call["loss"]) and torch.equal(stats, call["stats"])
    assert all(torch.equal(d.grad, g) for d, g in zip(ds, call["grads"]))
    assert call["grad_loss"].item() == 1.0
    _valid_somewhere({}, dbg)
    worst = PL.check_against_fp64(call["imgs"], call["pm"], call["depths"], call["dint"].reshape(-1),
                                  call["ratios"], 2, call["lam"], loss, stats, dbg, [d.grad for d in ds],
                                  "train 800x608")
    print(f"[photo train step] largest e error / bound {max(r for r, _ in worst):.3e}")


@pytest.mark.gpu
def test_photo_training_projections_match_cameras(textured_capture):
    """Ground-truth surface points of every training sample's reference view, warped through the
    sample's proj_mats at each level as the loss warps them (p = R (x, y, 1) + T / d in float64
    of the float32 matrices), land within 1e-3 px of their float64 projection by the COLMAP
    cameras scaled to the network size and the level."""
    ts = train_data.ColmapTrainSet(textured_capture, n_views=5, img_wh=TRAIN_WH, device=DEV, log=lambda *a: None)
    sc = ts.scan.scene

    def k_net(v):
        K = np.array(sc.K[v], np.float64).copy()
        K[0] *= TRAIN_WH[0] / sc.wh[v, 0]
        K[1] *= TRAIN_WH[1] / sc.wh[v, 1]
        return K

    worst, n = 0.0, 0
    for i, ids in enumerate(ts.ids):
        pm = ts.batch([i])["proj_mats"][0].double().cpu().numpy()        # (S, levels, 3, 4)
        depth, X = synth_scenes.height_field_depth(k_net(ids[0]), sc.E[ids[0]], TRAIN_WH)
        for l in range(3):
            d, Xl = depth[:: 1 << l, :: 1 << l], X[:: 1 << l, :: 1 << l]
            h, w = d.shape
            ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
            for s, v in enumerate(ids[1:]):
                E = np.asarray(sc.E[v], np.float64)
                q = np.einsum("ij,hwj->hwi", k_net(v), np.einsum("ij,hwj->hwi", E[:3, :3], Xl) + E[:3, 3])
                P = pm[s, l]
                p = np.einsum("ij,hwj->hwi", P[:, :3], np.stack([xs, ys, np.ones_like(xs)], -1)) \
                    + P[:, 3] / d[..., None]
                front = q[..., 2] > 0
                assert front.mean() > 0.5
                err = np.maximum(np.abs(p[..., 0] / p[..., 2] - q[..., 0] / q[..., 2] / (1 << l)),
                                 np.abs(p[..., 1] / p[..., 2] - q[..., 1] / q[..., 2] / (1 << l)))[front]
                worst = max(worst, float(err.max()))
                n += err.size
    print(f"[photo projections] {n} warps, largest error {worst:.3e} px")
    assert n > 0 and worst <= 1e-3


# ------------------------------------------------------------------------------------ SL1 loss
THRESHOLDS = (0.5, 1.0, 2.0, 4.0)
EPS32 = 2.0 ** -24
# name: W, H, B, levels, mask kind per level ("random": 80 % true, "true", "false")
SL1_CASES = {
    "640x512_b1": (640, 512, 1, 3, ("random",) * 3),
    "640x512_b2": (640, 512, 2, 3, ("random",) * 3),
    "640x512_b4": (640, 512, 4, 3, ("random",) * 3),
    "768x576_b4": (768, 576, 4, 3, ("random",) * 3),
    "1600x1184_b1": (1600, 1184, 1, 3, ("random",) * 3),
    "640x512_levels1": (640, 512, 2, 1, ("random",)),
    "640x512_levels2": (640, 512, 2, 2, ("random", "true")),
    "640x512_levels4": (640, 512, 2, 4, ("random",) * 4),
    "640x512_all_true": (640, 512, 2, 3, ("true",) * 3),
    "640x512_level1_empty": (640, 512, 2, 3, ("random", "false", "random")),
}


def sl1_inputs(W, H, B, levels, kinds, seed=0):
    """Per level float32 (pred, gt, mask) numpy arrays: gt in [520, 1000), so that pred - gt
    is exact in float32 (Sterbenz) for every difference used; differences ~ N(0, 2.5), with a
    quarter of the elements placed exactly at +-0.5, 1, 2 and 4."""
    rng = np.random.default_rng(seed)
    out = []
    for l in range(levels):
        shape = (B, H >> l, W >> l)
        gt = rng.uniform(520.0, 1000.0, shape).astype(np.float32)
        diff = rng.normal(0.0, 2.5, shape)
        exact = rng.random(shape) < 0.25
        diff[exact] = rng.choice(np.concatenate([THRESHOLDS, [-t for t in THRESHOLDS]]), exact.sum())
        pred = (gt.astype(np.float64) + diff).astype(np.float32)
        mask = {"random": rng.random(shape) < 0.8, "true": np.ones(shape, bool),
                "false": np.zeros(shape, bool)}[kinds[l]]
        out.append((pred, gt, mask))
    return out


def sl1_fp64(arrs):
    """(loss, [n_l], [sum |e|, #<1, #<2, #<4] of level 0 exactly, x per level) in float64 on the
    exact differences (NaN loss when a level's mask is empty, as 0/0)."""
    total, ns, xs = 0.0, [], []
    for l, (p, g, m) in enumerate(arrs):
        x = p.astype(np.float64) - g.astype(np.float64)
        xs.append(x)
        ax = np.abs(x[m])
        ns.append(int(m.sum()))
        s = math.fsum(np.where(ax < 1, 0.5 * ax * ax, ax - 0.5).tolist())
        total += 2.0 ** (1 - l) * (s / ns[-1] if ns[-1] else float("nan"))
    ax = np.abs(xs[0][arrs[0][2]])
    return total, ns, [math.fsum(ax.tolist()), int((ax < 1).sum()), int((ax < 2).sum()), int((ax < 4).sum())], xs


def aten_sl1_grad(pred, gt, mask, n, grad_loss, l):
    """ATen's gradient of smooth_l1_loss(p[m], g[m], reduction='mean') * 2^(1-l) in float32, one
    rounding per operation: go = grad * w, norm = (float)(1.0 / n); x <= -1: -norm * go,
    x >= 1: norm * go, else norm * x * go / beta (beta = 1); 0 off the mask."""
    f = np.float32
    go = f(grad_loss) * f(2.0 ** (1 - l))
    norm = f(1.0 / n) if n else f(np.inf)
    x = pred - gt
    with np.errstate(invalid="ignore"):
        r = np.where(x <= f(-1), -norm * go, np.where(x >= f(1), norm * go, (norm * x) * go / f(1)))
    return np.where(mask, r, f(0)).astype(np.float32)


def test_aten_sl1_grad_restatement_matches_torch():
    """The float32 restatement equals torch's CPU autograd of the reference's loss bit for bit,
    at 1, 3 and 4 levels, incoming gradients 1 and 0.37, exact threshold differences."""
    for levels, go in ((1, 1.0), (3, 1.0), (3, 0.37), (4, 0.37)):
        arrs = sl1_inputs(64, 48, 2, levels, ("random",) * levels, seed=levels)
        ps = [torch.from_numpy(p).requires_grad_(True) for p, _, _ in arrs]
        loss = sum(F.smooth_l1_loss(p[torch.from_numpy(m)], torch.from_numpy(g)[torch.from_numpy(m)],
                                    reduction="mean") * 2 ** (1 - l)
                   for l, (p, (_, g, m)) in enumerate(zip(ps, arrs)))
        loss.backward(torch.tensor(go))
        for l, (p, (pn, g, m)) in enumerate(zip(ps, arrs)):
            want = aten_sl1_grad(pn, g, m, int(m.sum()), go, l)
            assert np.array_equal(p.grad.numpy().view(np.int32), want.view(np.int32)), (levels, go, l)


def _f32_of_sum(got, exact):
    """got == float32(exact), or one ulp from it with exact within 1e-12 relative of the midpoint
    between the two (where a float64 sum in another order may round the other way)."""
    want = np.float32(exact)
    if got == want:
        return True
    mid = (float(got) + float(want)) / 2
    return (abs(np.float64(got) - np.float64(want)) == np.spacing(min(abs(got), abs(want)))
            and abs(exact - mid) <= 1e-12 * abs(exact))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SL1_CASES))
def test_sl1_vs_fp64(name):
    W, H, B, levels, kinds = SL1_CASES[name]
    arrs = sl1_inputs(W, H, B, levels, kinds, seed=len(name))
    l64, ns, m64, xs = sl1_fp64(arrs)
    for (p, g, _), x in zip(arrs, xs):
        assert np.array_equal((p - g).astype(np.float64), x)                     # the float32 difference is exact
    preds = {f"depth_{l}": torch.from_numpy(p).to(DEV).requires_grad_(True) for l, (p, _, _) in enumerate(arrs)}
    gts = {f"level_{l}": torch.from_numpy(g).to(DEV) for l, (_, g, _) in enumerate(arrs)}
    masks = {f"level_{l}": torch.from_numpy(m).to(DEV) for l, (_, _, m) in enumerate(arrs)}
    loss, metrics = losses.sl1_loss_and_metrics(preds, gts, masks, levels)
    go = 0.37
    loss.backward(torch.tensor(go, device=DEV))
    _, _, counts = losses._forward([preds[f"depth_{l}"] for l in range(levels)],
                                   [gts[f"level_{l}"] for l in range(levels)],
                                   [masks[f"level_{l}"] for l in range(levels)])
    assert counts.tolist() == ns
    lk = loss.item()
    if any(n == 0 for n in ns):
        assert math.isnan(lk) and math.isnan(l64)
    else:
        assert abs(lk - l64) <= np.spacing(np.float32(l64)), (lk, l64)
    m = metrics.cpu().numpy()
    assert m[1:4].tolist() == m64[1:4] and m[4] == ns[0]
    assert _f32_of_sum(m[0], m64[0]), (m[0], m64[0])
    for l, (p, g, mk) in enumerate(arrs):
        got = preds[f"depth_{l}"].grad.cpu().numpy()
        want = aten_sl1_grad(p, g, mk, ns[l], go, l)
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), f"level {l}"
        if ns[l]:
            # float64 derivative of the float32 incoming gradient; ATen rounds three times (1/n,
            # norm * x, * go; go * 2^(1-l) is exact), each within 2^-24 relative, so the error
            # is within 3 * 2^-24 of it (up to 2.2 float32 ulp: one ulp does not hold)
            d64 = np.where(mk, float(np.float32(go)) * 2.0 ** (1 - l) * np.clip(xs[l], -1, 1) / ns[l], 0.0)
            rel = np.abs(got - d64) / np.maximum(np.abs(d64), 1e-300)
            assert (rel <= 3 * EPS32 * (1 + 1e-6)).all(), (l, rel.max() / EPS32)
            worst_ulp = (np.abs(got - d64) / np.spacing(np.abs(d64).astype(np.float32))).max()
            print(f"[sl1 {name}] level {l}: gradient vs float64 at most {rel.max() / EPS32:.3f} x 2^-24 "
                  f"relative ({worst_ulp:.3f} float32 ulp)")
    dm = losses.depth_metrics(preds["depth_0"].detach(), gts["level_0"], masks["level_0"])
    assert torch.equal(dm, metrics)
    print(f"[sl1 {name}] loss {lk!r} vs fp64 {l64!r}, counts {ns}, metrics {m.tolist()}")
