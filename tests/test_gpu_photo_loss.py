"""The photometric loss (csrc/photo_loss.cu through losses.photo_loss) on the GPU:

  * per element against float64 (oracle/photo_loss_fp64.py, run in float64 on the device) at
    the level shapes of 640x512 (V = 3, K = 1) and 1152x864 (V = 5, K = 1..4), B = 2: validity,
    e within the oracle's bound, the selection wherever the oracle's margin exceeds twice its
    bound, loss_q, P_l, S_l, N_l and the loss, and the gradient given the kernel's selection;
  * two calls give the same bits; the call makes no host synchronisation;
  * the gradient is useful: Adam on the depth maps alone, from the ground truth of the textured
    capture plus a smooth perturbation of several depth intervals, halves the depth error;
  * train.main end to end with --dataset_name colmap --loss_type photo, its checkpoint through
    eval_pipeline --ckpt, a DTU run with photo logging the ground-truth metrics, and two
    --deterministic --seed runs writing the same bytes.
"""
import json
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import io, losses, synth, synth_scenes, train, train_data
from oracle import photo_loss_fp64 as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RATIOS = [1.0, 2.0, 4.0]
LAM = 0.1
EPS32 = 2.0 ** -24
# Share of (q, s) pairs whose validity may differ: a sample on the image border or at
# p_z = 1e-7 within float32's rounding of the warp; at most one pair per level was seen (4 over
# all cases), 2^-14 leaves room.  Pixels with such a pair are left out of the loss_q check.
VALID_MISMATCH_MAX = 2.0 ** -14
# Gradient: each element is a float32 sum of at most 9 windows x S sources x 3 channels of
# products of SSIM coefficients (quotients with denominators >= C1 C2) and bilinear slopes, so
# a few hundred ulp of the sum of the magnitudes, bounded here by 2^-10 of the element plus
# 2^-14 of the level's largest gradient.  Every pixel meets it except the oracle's kinks
# (LevelResult.kink: p's own warp within the warp bound of a tap-cell edge, where the bilinear
# slope differs between the precisions, or a sign of |x - y| or of a depth difference within
# rounding of 0) and the 3x3 neighbourhood of a window whose validity differs.  The kinks come
# from a worst-case warp bound, so they are a wide net (up to a fifth of the pixels at
# 1152x864 with 4 sources); the pixels actually out of tolerance, all of which must be kinks,
# were at most 2.0e-4 of a level, and may be at most 2^-12.
GRAD_REL, GRAD_ABS, OVER_SHARE_MAX = 2.0 ** -10, 2.0 ** -14, 2.0 ** -12


@pytest.fixture(autouse=True)
def _grad_mode():
    with torch.enable_grad():            # conftest runs GPU tests under no_grad by default
        yield


def make_case(B, V, W, H, seed=0):
    """Blurred-noise views (un-normalised in [0, 1]), the synthetic DTU projections, smooth
    depth maps around the views' convergence depth, different per level and sample."""
    rng = np.random.default_rng(seed)
    u8 = np.stack([cv2.GaussianBlur(rng.integers(0, 256, (H, W, 3), dtype=np.uint8), (0, 0), 2.0)
                   for _ in range(B * V)])
    imgs = io.normalize_images(torch.from_numpy(u8).to(DEV)).view(B, V, 3, H, W)
    pm = synth.projection_matrices(V, W, H, 3).unsqueeze(0).expand(B, -1, -1, -1, -1).contiguous().to(DEV)
    depths = []
    for l in range(3):
        ys, xs = np.mgrid[0:H >> l, 0:W >> l].astype(np.float64) * (1 << l)
        d = np.stack([synth.CONVERGE_MM + 40 * np.sin(xs / 37 + b) * np.cos(ys / 53) + 3 * l
                      + rng.normal(0, 0.5, xs.shape) for b in range(B)])
        depths.append(torch.from_numpy(d).float().to(DEV))
    dint = torch.tensor([[2.65], [3.1]][:B], device=DEV)
    return imgs, pm, depths, dint


def run(imgs, pm, depths, dint, K, debug=False):
    ds = [d.clone().requires_grad_(True) for d in depths]
    out = losses.photo_loss({f"depth_{l}": d for l, d in enumerate(ds)}, imgs, pm, dint, RATIOS, 3, K,
                            LAM, debug=debug)
    out[0].backward()
    return out, [d.grad for d in ds]


CASES = [(640, 512, 3, 1), (1152, 864, 5, 1), (1152, 864, 5, 2), (1152, 864, 5, 3), (1152, 864, 5, 4)]


@pytest.mark.parametrize("W,H,V,K", CASES)
def test_matches_float64(W, H, V, K):
    imgs, pm, depths, dint = make_case(2, V, W, H)
    (loss, stats, dbg), grads = run(imgs, pm, depths, dint, K, debug=True)
    with torch.no_grad():
        _, own = O.photo_loss(depths, imgs, pm, dint, RATIOS, K, LAM)
    sel = [k["selected"] & r.valid for k, r in zip(dbg, own)]
    L64, res, g64 = O.gradient(depths, imgs, pm, dint, RATIOS, K, LAM, selected=sel)
    tol_loss = 0.0
    for l, (k, r, rk) in enumerate(zip(dbg, own, res)):
        mism = (k["valid"] != r.valid).sum().item()
        assert mism <= VALID_MISMATCH_MAX * r.valid.numel(), (l, mism)
        both = k["valid"] & r.valid
        assert torch.isnan(k["e"][~k["valid"]]).all()
        err = (k["e"].double() - r.e).abs()[both]
        bound = r.e_bound[both]
        ratio = (err / bound).max().item()
        assert ratio <= 1.0, (l, ratio)
        qbound = torch.where(r.valid, r.e_bound, torch.zeros_like(r.e_bound)).amax(1)
        clear = (r.margin > 2 * qbound) & (k["valid"] == r.valid).all(1)
        assert torch.equal(k["selected"].permute(0, 2, 3, 1)[clear], r.selected.permute(0, 2, 3, 1)[clear])
        ambiguous = (~clear & (r.valid.sum(1) > K)).double().mean().item()
        same = (k["valid"] == r.valid).all(1)
        has = (rk.loss_q == rk.loss_q) & same
        assert torch.equal(has, (k["loss_q"] == k["loss_q"]) & same)
        lq_err = (k["loss_q"].double() - rk.loss_q).abs()[has]
        assert (lq_err <= qbound[has] + 4 * EPS32).all(), (l, lq_err.max().item())
        P, S, N = stats[l].double().tolist()
        assert N == rk.N.item() or mism, (l, N, rk.N.item())
        tolP = qbound.max().item() + 4 * EPS32
        assert abs(P - rk.P.item()) <= tolP, (l, P, rk.P.item())
        assert abs(S - rk.S.item()) <= 1e-5 * abs(rk.S.item()) + 1e-12, (l, S, rk.S.item())
        tol_loss += 2.0 ** (1 - l) * (tolP + LAM * 1e-5 * abs(rk.S.item()))
        g, gr = grads[l].double(), g64[l]
        scale = gr.abs().max().item()
        gerr = (g - gr).abs()
        over = gerr > GRAD_REL * gr.abs() + GRAD_ABS * scale
        moved = (k["valid"] != r.valid).any(1).double()[:, None]
        exempt = rk.kink | (torch.nn.functional.max_pool2d(moved, 3, 1, 1)[:, 0] > 0)
        bad = over & ~exempt
        assert not bad.any(), (l, bad.sum().item(), gerr[bad].max().item() / scale)
        share = over.double().mean().item()
        exempt_share = exempt.double().mean().item()
        assert share <= OVER_SHARE_MAX, (l, share)
        print(f"[photo {W}x{H} V={V} K={K} l={l}] e err/bound max {ratio:.3e}, e err max "
              f"{err.max().item():.3e}, loss_q err max {lq_err.max().item():.3e}, ambiguous "
              f"selection {ambiguous:.2e}, grad err max / level max {gerr.max().item() / scale:.3e}, "
              f"over tolerance {share:.2e} (all exempt; exempt share {exempt_share:.2e}), "
              f"validity mismatches {mism}")
    assert abs(loss.item() - L64.item()) <= tol_loss + 4 * EPS32 * abs(L64.item())


def test_level_without_valid_pixels():
    """Depths that put every sample behind the cameras: N_l = 0 and P_l = 0 at every level, so
    the backward's source loop never runs and the gradient is the smoothness term's alone.  It
    matches float64, two calls give the same bits, and a zero incoming gradient gives zeros."""
    imgs, pm, depths, dint = make_case(2, 3, 256, 192, seed=5)
    depths = [-d for d in depths]
    lam = 0.5
    outs = []
    for _ in range(2):
        ds = [d.clone().requires_grad_(True) for d in depths]
        loss, stats = losses.photo_loss({f"depth_{l}": d for l, d in enumerate(ds)}, imgs, pm, dint,
                                        RATIOS, 3, 1, lam)
        loss.backward()
        outs.append((loss, stats, [d.grad for d in ds]))
    (loss, stats, grads), (loss2, stats2, grads2) = outs
    assert torch.equal(loss, loss2) and torch.equal(stats, stats2)
    assert all(torch.equal(a, b) for a, b in zip(grads, grads2))
    assert (stats[:, 0] == 0).all() and (stats[:, 2] == 0).all()
    L64, res, g64 = O.gradient(depths, imgs, pm, dint, RATIOS, 1, lam)
    assert all(r.N.item() == 0 for r in res)
    assert abs(loss.item() - L64.item()) <= 1e-5 * abs(L64.item())
    for l, (g, gr, r) in enumerate(zip(grads, g64, res)):
        scale = gr.abs().max().item()
        assert scale > 0
        over = (g.double() - gr).abs() > GRAD_REL * gr.abs() + GRAD_ABS * scale
        assert not (over & ~r.kink).any(), l
    ds = [d.clone().requires_grad_(True) for d in depths]
    loss, _ = losses.photo_loss({f"depth_{l}": d for l, d in enumerate(ds)}, imgs, pm, dint, RATIOS, 3, 1, lam)
    (loss * 0).backward()
    assert all(torch.equal(d.grad, torch.zeros_like(d)) for d in ds)


def test_two_calls_same_bits_and_no_sync():
    imgs, pm, depths, dint = make_case(2, 5, 640, 512, seed=3)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        (l1, s1), g1 = run(imgs, pm, depths, dint, 2)
        (l2, s2), g2 = run(imgs, pm, depths, dint, 2)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(l1, l2) and torch.equal(s1, s2)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))


def test_refused_before_launch():
    imgs, pm, depths, dint = make_case(1, 3, 64, 64)
    res = {f"depth_{l}": d[:1] for l, d in enumerate(depths)}
    for kw in ({"topk": 0}, {"topk": 3}, {"smooth_weight": -1.0}, {"smooth_weight": float("inf")}):
        with pytest.raises(Exception, match="photo_loss_fwd"):
            losses.photo_loss(res, imgs, pm[:1], dint[:1], RATIOS, **kw)


# ------------------------------------------------------------------ the textured capture
@pytest.fixture(scope="module")
def capture(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("photo_capture"))
    synth_scenes.make_colmap(root, n_views=8, image_wh=(640, 512), n_points=3000, seed=5, textured=True)
    return root


def gt_depth(scene, v, img_wh):
    """Ground-truth depth of view v at the network size (its K scaled to img_wh)."""
    sc = scene.scan.scene
    K = sc.K[v].copy()
    K[0] *= img_wh[0] / sc.wh[v, 0]
    K[1] *= img_wh[1] / sc.wh[v, 1]
    return synth_scenes.height_field_depth(K, sc.E[v], img_wh)[0]


def test_gradient_recovers_depth(capture):
    wh = (640, 512)
    ts = train_data.ColmapTrainSet(capture, n_views=5, img_wh=wh, device=DEV)
    i = next(i for i, ids in enumerate(ts.ids) if ids[0] == 4)
    s = ts.batch([i])
    gt = torch.from_numpy(gt_depth(ts, 4, wh)).float().to(DEV)
    delta = s["depth_interval"].item()
    ys, xs = torch.meshgrid(torch.arange(wh[1], device=DEV), torch.arange(wh[0], device=DEV), indexing="ij")
    pert = 6 * delta * torch.sin(xs / 97.0) * torch.cos(ys / 71.0)
    start = gt + pert
    params = [start[None, :: 1 << l, :: 1 << l].clone().requires_grad_(True) for l in range(3)]
    opt = torch.optim.Adam(params, lr=0.1 * delta)
    before = (params[0].detach()[0] - gt).abs().mean().item()
    for _ in range(300):
        opt.zero_grad()
        # the photometric gradient alone
        loss, _ = losses.photo_loss({f"depth_{l}": p for l, p in enumerate(params)}, s["imgs"],
                                    s["proj_mats"], s["depth_interval"], RATIOS, smooth_weight=0.0)
        loss.backward()
        opt.step()
    after = (params[0].detach()[0] - gt).abs().mean().item()
    print(f"[photo adam] mean |depth - gt| at level 0: {before / delta:.3f} -> {after / delta:.3f} intervals")
    assert after <= 0.5 * before


def _train_argv(root, exp, *extra):
    return ["--dataset_name", "colmap", "--loss_type", "photo", "--root_dir", root, "--img_wh", "160",
            "128", "--n_views", "3", "--num_epochs", "1", "--log_every", "1", "--optimizer", "adam",
            "--exp_name", exp, *extra]


@pytest.fixture(scope="module")
def small_capture(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("photo_small"))
    synth_scenes.make_colmap(root, n_views=6, image_wh=(160, 128), n_points=2000, seed=2, textured=True)
    return root


def test_train_colmap_end_to_end(small_capture, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    trainer = train.main(_train_argv(small_capture, "tta"))
    recs = [json.loads(line) for line in open(tmp_path / "logs" / "tta" / "metrics.jsonl")]
    steps = [r for r in recs if "train/loss" in r]
    assert steps and trainer.global_step == 6
    for r in steps:
        assert all(np.isfinite(r[k]) for k in ("train/loss", "train/photo", "train/smooth"))
        assert "train/abs_err" not in r
    val = recs[-1]
    assert np.isfinite(val["val/loss"]) and val["checkpoint"]
    out = tmp_path / "out"
    ep.main(["--dataset_name", "colmap", "--root_dir", small_capture, "--out", str(out), "--img_wh", "160",
             "128", "--n_views", "3", "--ckpt", val["checkpoint"], "--conf", "0", "--min_geo_consistent", "0"])
    assert os.path.getsize(out / "points" / f"{os.path.basename(small_capture)}.ply") > 0


def test_train_dtu_photo_logs_ground_truth_metrics(tmp_path, monkeypatch):
    root = synth_scenes.make_dtu_train(str(tmp_path / "dtu"), seed=0)
    monkeypatch.chdir(tmp_path)
    train.main(["--root_dir", root, "--train_list", os.path.join(root, "lists", "train.txt"),
                "--val_list", os.path.join(root, "lists", "val.txt"), "--num_epochs", "1",
                "--log_every", "1", "--num_workers", "0", "--loss_type", "photo", "--photo_topk", "2",
                "--exp_name", "dtu_photo"])
    recs = [json.loads(line) for line in open(tmp_path / "logs" / "dtu_photo" / "metrics.jsonl")]
    step = next(r for r in recs if "train/loss" in r)
    for k in ("train/photo", "train/smooth", "train/abs_err", "train/acc_2mm"):
        assert np.isfinite(step[k]), k
    assert "val/acc_2mm" in recs[-1] and "val/photo" in recs[-1]


def test_two_deterministic_runs_write_the_same_bytes(small_capture, tmp_path):
    code = "import sys\nsys.path.insert(0, %r)\nfrom casmvsnet_pl_b200 import train\ntrain.main(sys.argv[1:])\n" % ROOT
    runs = []
    for i in range(2):
        cwd = tmp_path / f"run{i}"
        cwd.mkdir()
        subprocess.run([sys.executable, "-c", code] + _train_argv(small_capture, "det", "--deterministic",
                                                                  "--seed", "0"),
                       check=True, cwd=str(cwd), timeout=900)
        runs.append(cwd)
    logs = [open(r / "logs" / "det" / "metrics.jsonl", "rb").read() for r in runs]
    assert logs[0] and logs[0] == logs[1]
    names = sorted(os.listdir(runs[0] / "ckpts" / "det"))
    assert names and names == sorted(os.listdir(runs[1] / "ckpts" / "det"))
    for n in names:
        c0, c1 = (torch.load(r / "ckpts" / "det" / n, map_location="cpu") for r in runs)
        for k, v in c0["state_dict"].items():
            assert torch.equal(v, c1["state_dict"][k]), f"{n}: {k}"
