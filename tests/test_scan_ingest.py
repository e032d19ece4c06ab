"""Tanks and BlendedMVS scan readers and the resampler restatements, CPU tier.

The readers (eval_pipeline.TanksTestScan / BlendedMVSTestScan) with the host image route must
reproduce what the reference's TanksDataset / BlendedMVSDataset derived from the committed fixture
(tests/golden/scans, recorded by oracle/make_golden_scans.py), and the numpy restatements of
Pillow's BILINEAR and cv2's INTER_LINEAR resize (oracle/resize_oracle.py, and the weight tables
io.py uploads for the device kernels) must match the installed libraries byte for byte."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import io as cio
from oracle import resize_oracle as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "scans")

# (in W,H) -> (out W,H): the data sets' pairs, scaled-down versions, up-scales, one-axis and odd sizes
PAIRS = [((1600, 1200), (1152, 864)), ((1920, 1080), (1152, 864)), ((1920, 1080), (1920, 1056)),
         ((2048, 1080), (1920, 1056)), ((2048, 1536), (768, 576)), ((160, 120), (115, 86)),
         ((192, 108), (192, 105)), ((77, 50), (128, 96)), ((204, 108), (96, 64)),
         ((33, 17), (33, 40)), ((100, 80), (37, 80)), ((5, 4), (3, 7)), ((1, 5), (3, 2)),
         ((97, 61), (31, 29)), ((64, 48), (32, 24))]


def _img(W, H, seed):
    return np.random.default_rng(seed).integers(0, 256, (H, W, 3), dtype=np.uint8)


def _apply_pil_tables(img, wh):
    """io.pil_bilinear_coeffs applied as the kernel applies them."""
    t = img.astype(np.int64)
    for axis, n in ((1, wh[0]), (0, wh[1])):
        if n == t.shape[axis]:
            continue
        b, k = cio.pil_bilinear_coeffs(t.shape[axis], n)
        a = np.moveaxis(t, axis, 0)
        out = np.empty((n,) + a.shape[1:], np.int64)
        for o in range(n):
            s = np.full(a.shape[1:], 1 << 21, np.int64)
            for j in range(b[o, 1]):
                s += a[b[o, 0] + j] * k[o, j]
            out[o] = np.clip(s >> 22, 0, 255)
        t = np.moveaxis(out, 0, axis)
    return t.astype(np.uint8)


def _apply_cv_tables(img, wh):
    xt = cio.cv2_linear_table(img.shape[1], wh[0], True).astype(np.int64)
    yt = cio.cv2_linear_table(img.shape[0], wh[1], False).astype(np.int64)
    I = img.astype(np.int64)
    rows = I[:, xt[:, 0]] * xt[None, :, 2, None] + I[:, xt[:, 1]] * xt[None, :, 3, None]
    v = (((rows[yt[:, 0]] >> 4) * yt[:, 2, None, None]) >> 16) + \
        (((rows[yt[:, 1]] >> 4) * yt[:, 3, None, None]) >> 16)
    return ((v + 2) >> 2).astype(np.uint8)


@pytest.mark.parametrize("pair", PAIRS[5:])
def test_pil_restatement_matches_pillow(pair):
    from PIL import Image
    (W, H), wh = pair
    img = _img(W, H, W * 7 + H)
    ref = np.asarray(Image.fromarray(img).resize(wh, Image.BILINEAR))
    assert np.array_equal(R.pil_bilinear(img, wh), ref)
    assert np.array_equal(_apply_pil_tables(img, wh), ref)


@pytest.mark.parametrize("pair", PAIRS)
def test_cv2_restatement_matches_opencv(pair):
    cv2 = pytest.importorskip("cv2")
    (W, H), wh = pair
    img = _img(W, H, W * 5 + H)
    ref = cv2.resize(img, wh, interpolation=cv2.INTER_LINEAR)
    assert np.array_equal(R.cv2_linear(img, wh), ref)
    assert np.array_equal(_apply_cv_tables(img, wh), ref)


def test_pil_restatement_matches_pillow_at_dataset_sizes():
    """The full-size pairs once each (the per-output Python loop is slow at 1920 wide)."""
    from PIL import Image
    for (W, H), wh in PAIRS[:5]:
        img = _img(W, H, 3)
        ref = np.asarray(Image.fromarray(img).resize(wh, Image.BILINEAR))
        assert np.array_equal(_apply_pil_tables(img, wh), ref), ((W, H), wh)


def _normalize_cpu(u8):
    """ToTensor + Normalize (datasets/tanks.py:114-118) on the host."""
    x = torch.from_numpy(u8).permute(0, 3, 1, 2).float().div(255)
    mean = torch.tensor(cio.IMAGENET_MEAN)[:, None, None]
    std = torch.tensor(cio.IMAGENET_STD)[:, None, None]
    return x.sub(mean).div(std)


def _check_scan_against_golden(scan, g):
    assert [r for r, _ in scan.metas] == g["ref"].tolist()
    for (ref, srcs), m in zip(scan.metas, g["metas"]):
        assert [ref] + srcs == [v for v in m.tolist() if v >= 0]
    for i, v in enumerate(g["view_ids"]):
        assert torch.equal(scan.proj_mats[int(v)], torch.from_numpy(g["view_proj"][i]))
        assert scan.depth_min[int(v)] == g["view_depth_min"][i]
    for i, (ref, srcs) in enumerate(scan.metas):
        ids = [ref] + srcs[: scan.n_views - 1]
        pm = cio.relative_proj_mats(scan.proj_mats, ids)
        assert torch.equal(pm, torch.from_numpy(g["proj_mats"][i]))
        dmin, dint = scan.depth_range(ref, 2.65)
        assert dmin == g["init_depth_min"][i] and dint == g["depth_interval"][i]
        u8 = np.stack([ep.read_network_image_u8(scan.image_path(v), scan.img_wh) for v in ids])
        assert torch.equal(_normalize_cpu(u8), torch.from_numpy(g["imgs"][i]))


def test_tanks_reader_matches_reference_golden():
    g = dict(np.load(os.path.join(GOLDEN, "tanks.npz")))
    scan = ep.TanksTestScan(os.path.join(GOLDEN, "tanks"), "intermediate", "Family",
                            tuple(g["img_wh"]), int(g["n_views"]), host_images=True)
    _check_scan_against_golden(scan, g)
    assert scan.depth_range(0, 123.0)[1] == np.float32(2.5e-3)     # --depth_interval has no effect


def test_blendedmvs_reader_matches_reference_golden():
    g = dict(np.load(os.path.join(GOLDEN, "blendedmvs.npz")))
    root = os.path.join(GOLDEN, "blendedmvs", "dataset_low_res")
    assert ep.BlendedMVSTestScan.scans(root, "val") == ["5a3ca9cb270f0e3f14d0eddb"]
    scan = ep.BlendedMVSTestScan(root, "5a3ca9cb270f0e3f14d0eddb", tuple(g["img_wh"]),
                                 int(g["n_views"]), float(g["n_depths_arg"]), host_images=True)
    assert scan.full_wh == (768, 576)
    assert scan.scale_factor == g["scale_factor"]
    assert len(scan.metas) < len(g["view_ids"])                      # views with 2 sources skipped
    _check_scan_against_golden(scan, g)


def test_unknown_tanks_scan_is_rejected():
    with pytest.raises(ValueError):
        ep.TanksTestScan(os.path.join(GOLDEN, "tanks"), "intermediate", "NoSuchScan", (64, 32), 3)


def test_cli_rejects_bad_split_and_dtu_gt(tmp_path):
    with pytest.raises(SystemExit):
        ep.main(["--root_dir", str(tmp_path), "--dataset_name", "tanks", "--split", "test"])
    with pytest.raises(SystemExit):
        ep.main(["--root_dir", str(tmp_path), "--dataset_name", "blendedmvs", "--split", "x"])
    with pytest.raises(SystemExit):
        ep.main(["--root_dir", str(tmp_path), "--dataset_name", "tanks", "--dtu_gt", "g"])


def test_save_visual_writes_reference_jpegs(tmp_path):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    depth = rng.uniform(400, 900, (32, 64)).astype(np.float32)
    depth[:4] = 0
    proba = rng.uniform(0, 1, (8, 16)).astype(np.float32)
    cio.save_visual(str(tmp_path), "s", 3, depth, proba, 0.5)
    d = cv2.imread(str(tmp_path / "s" / "depth_visual_0003.jpg"))
    p = cv2.imread(str(tmp_path / "s" / "proba_visual_0003.jpg"), cv2.IMREAD_GRAYSCALE)
    assert d.shape == (32, 64, 3) and p.shape == (8, 16)
