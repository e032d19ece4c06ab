"""The photometric loss without a GPU: the float64 oracle's gradient against central
differences, every refusal (the kernel entry's, before any device work, and train.py's), the
textured synthetic capture's photo-consistency under its ground-truth depth, and make_colmap's
untextured bytes."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch
from PIL import Image

from casmvsnet_pl_b200 import _lib, colmap, io, synth_scenes, train
from oracle import photo_loss_fp64 as O

RATIOS = [1.0, 2.0, 4.0]


def capture_case(root, wh=(96, 64), views=(0, 2, 4), seed=0):
    """The textured capture's even (same-size PINHOLE) views as a loss input on the CPU."""
    _, depths = synth_scenes.make_colmap(root, n_views=8, image_wh=wh, seed=seed, textured=True)
    sc = colmap.load_scene(root)
    pm = {v: io.pyramid_proj_mats(sc.K[v].astype(np.float32), sc.E[v].astype(np.float32), 3, wh, wh)
          for v in views}
    u8 = np.stack([np.array(Image.open(os.path.join(root, "images", sc.names[v]))) for v in views])
    x = torch.from_numpy(u8).permute(0, 3, 1, 2).double() / 255
    mean = torch.tensor(O.MEAN, dtype=torch.float64).view(3, 1, 1)
    std = torch.tensor(O.STD, dtype=torch.float64).view(3, 1, 1)
    imgs = ((x - mean) / std).float()[None]
    gt = torch.from_numpy(depths[views[0]]).float()
    return imgs, io.relative_proj_mats(pm, list(views))[None], gt


def levels_of(d):
    return [d[None, :: 1 << l, :: 1 << l].contiguous() for l in range(3)]


def test_textured_capture_is_photo_consistent(tmp_path):
    imgs, pm, gt = capture_case(str(tmp_path))
    dint = torch.tensor([0.01])
    L0, r0 = O.photo_loss(levels_of(gt), imgs, pm, dint, RATIOS, 1, 0.0)
    assert all(r.N > 0 for r in r0)
    # under the true depth the warped views agree to 8-bit quantisation and resampling
    assert r0[0].P < 2e-3, [float(r.P) for r in r0]
    for f in (0.97, 1.03):
        L1, _ = O.photo_loss(levels_of(gt * f), imgs, pm, dint, RATIOS, 1, 0.0)
        assert L1 > 1.5 * L0, (f, float(L0), float(L1))


def test_oracle_gradient_matches_central_differences(tmp_path):
    imgs, pm, gt = capture_case(str(tmp_path), wh=(64, 64))
    dint = torch.tensor([0.01])
    rng = np.random.default_rng(0)
    ds = [d.double() + 0.02 * torch.from_numpy(rng.standard_normal(d.shape)) for d in levels_of(gt)]
    for K, lam in ((1, 0.1), (2, 0.5)):
        _, res, grads = O.gradient(ds, imgs, pm, dint, RATIOS, K, lam)
        checked = 0
        for l in range(3):
            h = 1e-6
            for _ in range(40):
                y, x = (int(rng.integers(2, n - 2)) for n in ds[l].shape[1:])
                vals = []
                for step in (-h, 0.0, h):
                    dd = [d.clone() for d in ds]
                    dd[l][0, y, x] += step
                    with torch.no_grad():
                        vals.append(float(O.photo_loss(dd, imgs, pm, dint, RATIOS, K, lam)[0]))
                left, right = (vals[1] - vals[0]) / h, (vals[2] - vals[1]) / h
                if abs(left - right) > 1e-4 * max(abs(left), abs(right), 1e-9):
                    continue        # a kink (tap cell edge, top-K swap, |.| at 0) is in reach
                central = (vals[2] - vals[0]) / (2 * h)
                g = float(grads[l][0, y, x])
                assert abs(g - central) <= 1e-5 * abs(central) + 1e-9, (K, l, y, x, g, central)
                checked += 1
        assert checked >= 60, checked


def test_make_colmap_untextured_bytes_unchanged(tmp_path):
    synth_scenes.make_colmap(str(tmp_path), image_ext="png", fmt="both", seed=3)
    h = hashlib.sha256()
    for dp, _, fs in sorted(os.walk(tmp_path)):
        for f in sorted(fs):
            p = os.path.join(dp, f)
            h.update(os.path.relpath(p, tmp_path).encode())
            h.update(open(p, "rb").read())
    assert h.hexdigest() == "57c3ece84b8388b08d13ee052d6eefa4ca3b2adb83204a5088557e6f09f77f5f"


def test_kernel_entry_refuses_before_launch():
    lib = _lib.load()
    ok = ctypes.c_void_p(0x10000)
    ptrs = (ctypes.c_void_p * 4)(*([0x10000] * 4))
    ratios = (ctypes.c_float * 4)(1.0, 2.0, 4.0, 8.0)

    def fwd(V=3, H=64, W=64, levels=3, K=1, lam=0.1):
        return lib.casmvs_photo_loss_fwd(ok, ok, ok, ptrs, ratios, 1, V, H, W, levels, K, lam, ptrs, ok, ok,
                                         ok, None, None, None, ok, 1 << 20, None)

    def bwd(V=3, H=64, W=64, levels=3, K=1, lam=0.1):
        return lib.casmvs_photo_loss_bwd(ok, ok, ok, ptrs, ratios, 1, V, H, W, levels, K, lam, ptrs, ok, ok,
                                         ptrs, None)
    cases = [dict(V=1), dict(V=18), dict(K=0), dict(K=3), dict(V=5, K=5), dict(levels=5), dict(levels=0),
             dict(H=8, W=64), dict(H=64, W=8), dict(lam=-0.5), dict(lam=float("nan")),
             dict(lam=float("inf"))]
    for kw in cases:
        for entry in (fwd, bwd):
            assert entry(**kw) == -1, kw
            assert lib.casmvs_last_error(), kw
    assert lib.casmvs_photo_loss_workspace_bytes(2, 512, 640, 3) > 0


@pytest.mark.parametrize("argv,message", [
    (["--dataset_name", "colmap"], "--loss_type photo"),
    (["--dataset_name", "colmap", "--loss_type", "photo", "--train_list", "x"], "--train_list"),
    (["--dataset_name", "colmap", "--loss_type", "photo", "--val_list", "x"], "--val_list"),
    (["--img_wh", "640", "512", "--train_list", "a", "--val_list", "b"], "--img_wh"),
    (["--dataset_name", "blendedmvs", "--loss_type", "photo"], "blendedmvs"),
    (["--photo_topk", "1", "--train_list", "a", "--val_list", "b"], "--photo_topk"),
    (["--smooth_weight", "0.2", "--train_list", "a", "--val_list", "b"], "--smooth_weight"),
    (["--loss_type", "photo", "--photo_topk", "3", "--train_list", "a", "--val_list", "b"], "--photo_topk"),
    (["--loss_type", "photo", "--photo_topk", "0", "--train_list", "a", "--val_list", "b"], "--photo_topk"),
    (["--loss_type", "photo", "--smooth_weight", "-1", "--train_list", "a", "--val_list", "b"], "--smooth_weight"),
    (["--dataset_name", "colmap", "--loss_type", "photo", "--img_wh", "100", "64"], "--img_wh"),
])
def test_train_refusals(argv, message):
    with pytest.raises(SystemExit, match=message):
        train.check_supported(train.parse_args(argv))


def test_train_flags_resolve_per_data_set():
    a = train.parse_args(["--dataset_name", "colmap", "--loss_type", "photo"])
    train.check_supported(a)
    assert a.depth_interval == 192.0 and train.option(a, "img_wh") == [640, 512]
    assert train.option(a, "photo_topk") == 1 and train.option(a, "smooth_weight") == 0.01
    assert train.parse_args([]).depth_interval == 2.65
    a = train.parse_args(["--loss_type", "photo", "--n_views", "5", "--photo_topk", "4",
                          "--smooth_weight", "0", "--train_list", "a", "--val_list", "b"])
    train.check_supported(a)
    assert (a.photo_topk, a.smooth_weight) == (4, 0.0)
