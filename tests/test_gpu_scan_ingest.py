"""Device image ingest of the Tanks and BlendedMVS scan readers (GPU tier).

csrc/resize.cu must be byte-identical to Pillow's BILINEAR and cv2's INTER_LINEAR resize, the
cached network input of a reference view bit-identical to ToTensor + Normalize of the PIL-resized
image, and a whole scan through run_scan must give the same depth maps, confidence maps and PLY
bytes with the device image route as with the reference's host PIL / cv2 route."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib
from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import io as cio

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "scans")

PAIRS = [((1600, 1200), (1152, 864)), ((1920, 1080), (1152, 864)), ((1920, 1080), (1920, 1056)),
         ((2048, 1080), (1920, 1056)), ((768, 576), (768, 576)), ((2048, 1536), (768, 576)),
         ((77, 50), (128, 96)), ((97, 61), (31, 29)), ((33, 17), (33, 40)), ((100, 80), (37, 80)),
         ((5, 4), (3, 7))]


def _imgs(N, W, H, seed):
    return np.random.default_rng(seed).integers(0, 256, (N, H, W, 3), dtype=np.uint8)


@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("pair", PAIRS)
def test_resize_kernels_are_byte_identical_to_pillow_and_cv2(pair, N):
    import cv2
    from PIL import Image
    (W, H), wh = pair
    host = _imgs(N, W, H, W + H + N)
    dev = torch.from_numpy(host).cuda()
    pil = cio.resize_u8_pil(dev, wh).cpu().numpy()
    lin = cio.resize_u8_linear(dev, wh).cpu().numpy()
    for i in range(N):
        assert np.array_equal(pil[i], np.asarray(Image.fromarray(host[i]).resize(wh, Image.BILINEAR)))
        assert np.array_equal(lin[i], cv2.resize(host[i], wh, interpolation=cv2.INTER_LINEAR))


def test_resize_argument_validation():
    x = torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device="cuda")
    for bad in (x.cpu(), x.float(), x[..., :2], x[0]):
        with pytest.raises(_lib.CasMVSError):
            cio.resize_u8_pil(bad, (4, 4))
        with pytest.raises(_lib.CasMVSError):
            cio.resize_u8_linear(bad, (4, 4))
    for wh in ((0, 4), (4, -1)):
        with pytest.raises(_lib.CasMVSError):
            cio.resize_u8_pil(x, wh)
        with pytest.raises(_lib.CasMVSError):
            cio.resize_u8_linear(x, wh)
    lib = _lib.load()
    p = x.data_ptr()
    # null images, missing x tables for a horizontal pass, missing tmp for two passes
    assert lib.casmvs_resize_u8_pil_fwd(None, p, None, 1, 8, 8, 4, 8, None, None, 0, p, p, 3, None) != 0
    assert lib.casmvs_resize_u8_pil_fwd(p, p, None, 1, 8, 8, 8, 4, None, None, 0, None, None, 0, None) != 0
    assert lib.casmvs_resize_u8_pil_fwd(p, p, None, 1, 8, 8, 4, 4, p, p, 3, p, p, 3, None) != 0
    assert lib.casmvs_resize_u8_linear_fwd(p, p, 1, 8, 8, 0, 4, p, p, None) != 0
    assert lib.casmvs_resize_u8_linear_fwd(p, p, 1, 8, 8, 4, 4, p + 4, p, None) != 0


def test_cached_network_input_equals_reference_golden():
    """SceneImages gather + normalise == the reference's ToTensor + Normalize of the PIL resize,
    recorded from TanksDataset / BlendedMVSDataset; BlendedMVS depth intervals == golden."""
    g = dict(np.load(os.path.join(GOLDEN, "tanks.npz")))
    scan = ep.TanksTestScan(os.path.join(GOLDEN, "tanks"), "intermediate", "Family",
                            tuple(g["img_wh"]), int(g["n_views"]))
    for i, (ref, imgs, pm) in enumerate(scan.views("cuda:0")):
        assert torch.equal(imgs.cpu(), torch.from_numpy(g["imgs"][i]))
        assert torch.equal(pm, torch.from_numpy(g["proj_mats"][i]))
    g = dict(np.load(os.path.join(GOLDEN, "blendedmvs.npz")))
    scan = ep.BlendedMVSTestScan(os.path.join(GOLDEN, "blendedmvs", "dataset_low_res"),
                                 "5a3ca9cb270f0e3f14d0eddb", tuple(g["img_wh"]), int(g["n_views"]),
                                 float(g["n_depths_arg"]))
    seen = []
    for i, (ref, imgs, pm) in enumerate(scan.views("cuda:0")):
        assert torch.equal(imgs.cpu(), torch.from_numpy(g["imgs"][i]))
        assert scan.depth_range(ref, 2.65) == (g["init_depth_min"][i], g["depth_interval"][i])
        seen.append(ref)
    assert seen == g["ref"].tolist()


def _model(precision):
    from casmvsnet_pl_b200 import ABN, synth
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN, precision=precision)
    synth.randomize_model_(model, 0)
    return model.eval().cuda()


def _run(model, scan, tmp, tag):
    xyz, rgb = ep.run_scan(model, scan, conf=0.0, min_geo_consistent=0,
                           depth_dir=str(tmp / tag / "depth"), ply_path=str(tmp / tag / "s.ply"))
    d = tmp / tag / "depth" / scan.scan
    maps = {f: cio.read_pfm(d / f)[0] for f in sorted(os.listdir(d))}
    return maps, (tmp / tag / "s.ply").read_bytes(), len(xyz)


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
def test_scans_end_to_end_device_ingest_equals_host_route(tmp_path, precision):
    from casmvsnet_pl_b200 import synth_scenes
    model = _model(precision)
    n0 = _lib.fallback_count()
    tanks = synth_scenes.make_tanks(str(tmp_path / "tnt"), "intermediate", "Horse", n_views=6,
                                    image_wh=(200, 120), seed=3)
    assert os.path.isdir(tanks)
    bm_root = synth_scenes.make_blendedmvs(str(tmp_path / "bmvs"), "scanA", n_views=7,
                                           image_wh=(192, 144), seed=4, n_few=3)
    mk = {
        "tanks": lambda host: ep.TanksTestScan(str(tmp_path / "tnt"), "intermediate", "Horse",
                                               (160, 128), 3, host_images=host),
        "bmvs": lambda host: ep.BlendedMVSTestScan(bm_root, "scanA", (160, 128), 3, 2.65,
                                                   host_images=host),
    }
    for name, make in mk.items():
        dev_maps, dev_ply, n_dev = _run(model, make(False), tmp_path, f"{name}_dev_{precision}")
        host_maps, host_ply, _ = _run(model, make(True), tmp_path, f"{name}_host_{precision}")
        assert dev_maps.keys() == host_maps.keys()
        for k in dev_maps:
            assert np.array_equal(dev_maps[k], host_maps[k]), (name, k)
        assert dev_ply == host_ply and n_dev > 0
        scan = make(False)
        refs = sorted(r for r, _ in scan.metas)
        assert sorted({int(k[6:10]) for k in dev_maps}) == refs
        if name == "bmvs":          # views 2 and 5 list 2 sources < n_views = 3: skipped
            assert refs == [0, 1, 3, 4, 6]
        else:
            assert refs == list(range(6))
    assert _lib.fallback_count() == n0


def test_cli_writes_a_ply_per_scan(tmp_path):
    from casmvsnet_pl_b200 import synth_scenes
    for i, s in enumerate(ep.TanksTestScan.SCANS["intermediate"]):
        synth_scenes.make_tanks(str(tmp_path / "tnt"), "intermediate", s, n_views=3,
                                image_wh=(120, 70), seed=i)
    common = ["--img_wh", "64", "64", "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0"]
    ep.main(["--dataset_name", "tanks", "--split", "intermediate", "--root_dir", str(tmp_path / "tnt"),
             "--out", str(tmp_path / "out_t"), "--save_visual"] + common)
    for s in ep.TanksTestScan.SCANS["intermediate"]:
        assert os.path.getsize(tmp_path / "out_t" / "points" / f"{s}.ply") > 0
    assert os.path.isfile(tmp_path / "out_t" / "depth" / "Family" / "depth_visual_0000.jpg")
    root = None
    for i, s in enumerate(("scanA", "scanB")):
        root = synth_scenes.make_blendedmvs(str(tmp_path / "bm"), s, n_views=4, image_wh=(96, 72),
                                            seed=i, n_few=0, lists=("all",))
    ep.main(["--dataset_name", "blendedmvs", "--split", "all", "--root_dir", root,
             "--out", str(tmp_path / "out_b")] + common)
    for s in ("scanA", "scanB"):
        assert os.path.getsize(tmp_path / "out_b" / "points" / f"{s}.ply") > 0
