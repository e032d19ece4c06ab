"""BlendedMVS training, host side: the training reader against goldens recorded from the
reference's BlendedMVSDataset (oracle/make_golden_train_blendedmvs.py ->
tests/golden/train/blendedmvs_reader.npz, on the committed fixture tests/golden/train/blendedmvs),
its ColorJitter draws, the numpy jitter oracle against Pillow, and the trainer's arguments.
CPU only."""
import hashlib
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import train, train_data
from oracle import jitter_oracle as J
from oracle.make_golden_train_blendedmvs import FIXTURE_ROOT, N_DEPTHS_ARG, SEED

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train")


def _golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return {k: z[k] for k in z.files}


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("split", ["train", "val"])
def test_reader_matches_reference(split):
    g = _golden("blendedmvs_reader")
    p = split + "/"
    ds = train_data.BlendedMVSTrainDataset(FIXTURE_ROOT, split, 3, 3, N_DEPTHS_ARG)
    assert len(ds) == len(g[p + "metas"])
    assert [ds.scale_factors[s] for s in ds.scans] == g[p + "scale_factors"].tolist()
    assert sorted((s, str(v)) for s in ds.scans for v in ds.proj_mats[s]) == \
        sorted(map(tuple, g[p + "ref_views"].tolist())), "every pair.txt view has projections"
    order = list(g["digest_order"])
    for i, (scan, _, ref, srcs) in enumerate(ds.metas):
        assert scan == g[p + "scans"][i] and [ref] + srcs == g[p + "metas"][i].tolist()
        torch.manual_seed(int(SEED) + i)
        s = ds[i]
        assert _sha(torch.get_rng_state().numpy()) == g[p + "rng_after"][i], (i, "RNG consumption")
        assert s["scan_vid"] == (scan, ref)
        assert np.array_equal(s["proj_mats"].numpy(), g[p + "proj_mats"][i])
        assert np.array_equal(s["init_depth_min"].numpy(), g[p + "init_depth_min"][i])
        assert np.array_equal(s["depth_interval"].numpy(), g[p + "depth_interval"][i])
        assert s["imgs_u8"].shape == (3, 576, 768, 3) and s["imgs_u8"].dtype == torch.uint8
        for l in range(3):
            d, m = s["depths"][f"level_{l}"], s["masks"][f"level_{l}"]
            assert d.shape == (576 >> l, 768 >> l) and m.dtype == torch.bool
            assert _sha(d.numpy()) == g[p + "digests"][i][order.index(f"depth_{l}")], (i, l)
            assert _sha(m.numpy()) == g[p + "digests"][i][order.index(f"mask_{l}")], (i, l)
        assert (split == "train") == ("jitter" in s)
        # the images through the host oracle of the device transform: the reference's bits
        u8 = s["imgs_u8"].numpy()
        imgs = J.jitter_normalize(u8, s["jitter"].numpy()) if "jitter" in s else \
            np.stack([J.normalize(im) for im in u8])
        assert _sha(imgs) == g[p + "digests"][i][order.index("imgs")], i


def test_reader_skips_views_with_few_sources():
    ds = train_data.BlendedMVSTrainDataset(FIXTURE_ROOT, "all", 3, 3, N_DEPTHS_ARG)
    refs = {(s, r) for s, _, r, _ in ds.metas}
    assert all(r % 4 != 3 for _, r in refs) and len(refs) == 11
    assert "jitter" not in ds[0]                          # only the train split is jittered
    with pytest.raises(ValueError):
        train_data.BlendedMVSTrainDataset(FIXTURE_ROOT, "test")


def test_draws_equal_colorjitter_get_params():
    from torchvision import transforms as T
    cj = T.ColorJitter(brightness=0.25, contrast=0.5)
    for seed in range(20):
        torch.manual_seed(seed)
        ours = [train_data.draw_jitter() for _ in range(3)]
        torch.manual_seed(seed)
        for bf, b, c in ours:
            order, rb, rc, rs, rh = cj.get_params(cj.brightness, cj.contrast, None, None)
            order = order.tolist()
            assert (bf == 1.0) == (order.index(0) < order.index(1))
            assert (b, c, rs, rh) == (rb, rc, None, None)
            assert np.float32(b) == b and np.float32(c) == c    # exact float32 values


def _alphas():
    out = []
    for a in (0.5, 0.75, 1.0, 1.25, 1.5):
        f = np.float32(a)
        out += [f, np.nextafter(f, np.float32(0)), np.nextafter(f, np.float32(2))]
    rng = np.random.default_rng(0)
    out += list(rng.uniform(0.5, 1.5, 12).astype(np.float32)) + [np.float32(0.0), np.float32(2.0)]
    return out


def test_blend_oracle_matches_pillow_exhaustively():
    """Every (in1, in2) byte pair, for alphas on both of Blend.c's branches."""
    from PIL import Image
    in1, in2 = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    im1, im2 = Image.fromarray(np.ascontiguousarray(in1)), Image.fromarray(np.ascontiguousarray(in2))
    for a in _alphas():
        want = np.asarray(Image.blend(im1, im2, float(a)))
        assert np.array_equal(J.pil_blend(in1, in2, a), want), float(a)


def test_luma_oracle_matches_pillow_on_every_rgb_triple():
    from PIL import Image
    rgb = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(rgb >> 16) & 255, (rgb >> 8) & 255, rgb & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    want = np.asarray(Image.fromarray(img).convert("L"))
    assert np.array_equal(J.pil_luma(img), want)


def test_contrast_mean_and_jitter_match_pillow():
    from PIL import Image, ImageStat
    from torchvision.transforms import functional as F
    rng = np.random.default_rng(1)
    for k in range(40):
        h, w = rng.integers(1, 60, 2)
        lo, hi = sorted(rng.integers(0, 256, 2))
        img = rng.integers(lo, hi + 1, (h, w, 3), dtype=np.uint8)
        im = Image.fromarray(img)
        assert J.contrast_mean(img) == int(ImageStat.Stat(im.convert("L")).mean[0] + 0.5)
        bf = bool(k % 2)
        b, c = float(np.float32(rng.uniform(0.75, 1.25))), float(np.float32(rng.uniform(0.5, 1.5)))
        want = im
        for fn in (("b", "c") if bf else ("c", "b")):
            want = F.adjust_brightness(want, b) if fn == "b" else F.adjust_contrast(want, c)
        assert np.array_equal(J.jitter_u8(img, bf, b, c), np.asarray(want)), k


def test_jitter_golden_matches_oracle():
    g = _golden("jitter")
    for i, (k, j) in enumerate(zip(g["image_index"], g["jitter"])):
        out = J.jitter_u8(g["images"][k], bool(j[0]), float(j[1]), float(j[2]))
        assert np.array_equal(out, g["jittered"][i]), (i, j)
        assert _sha(J.normalize(out)) == g["normalized_sha"][i]
    for i, j in enumerate(g["odd_jitter"]):
        assert np.array_equal(J.jitter_u8(g["odd_image"], bool(j[0]), float(j[1]), float(j[2])),
                              g["odd_jittered"][i])
    sat = g["jittered"]
    assert (sat == 0).any() and (sat == 255).any()


def _check(argv):
    a = train.build_parser().parse_args(argv)
    train.check_supported(a)
    return a


def test_cli_accepts_blendedmvs_and_rejects_lists():
    a = _check(["--dataset_name", "blendedmvs", "--depth_interval", "192.0"])
    assert a.dataset_name == "blendedmvs" and a.depth_interval == 192.0
    for flag in ("--train_list", "--val_list"):
        with pytest.raises(SystemExit) as e:
            _check(["--dataset_name", "blendedmvs", flag, "x"])
        assert flag in str(e.value.code)
    with pytest.raises(SystemExit) as e:
        _check(["--dataset_name", "dtu"])
    assert "--train_list" in str(e.value.code)
    _check(["--train_list", "x", "--val_list", "y"])
    with pytest.raises(SystemExit):
        _check(["--dataset_name", "blendedmvs", "--use_amp"])
