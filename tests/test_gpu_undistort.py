"""Undistortion on the GPU: casmvs_undistort_u8_fwd against the float64 oracle for every model,
the identity at zero coefficients, the direction of the map on an analytic texture, and
eval_pipeline --dataset_name colmap on a distorted mapper project against the pinhole route on
the same views undistorted."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, colmap, io as cio, synth_scenes
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import undistort_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# coefficients of each model for a camera of width W (focal length and principal point scale)
COEFFS = {
    "SIMPLE_RADIAL": [-0.12], "RADIAL": [-0.15, 0.04],
    "OPENCV": [-0.21, 0.05, 1.2e-3, -8e-4],
    "FULL_OPENCV": [0.35, -0.1, 1.2e-3, -8e-4, 0.02, 0.55, -0.05, 0.01],
    "SIMPLE_RADIAL_FISHEYE": [0.03], "RADIAL_FISHEYE": [0.03, -0.01],
    "OPENCV_FISHEYE": [0.04, -0.012, 0.003, -0.0004],
}


def _params(model, w, h, coeffs):
    f = (0.47 if model in O.FISHEYE else 0.81) * w
    focal = [f] if model in O.SINGLE_FOCAL else [f, 1.013 * f]
    return focal + [0.497 * w + 0.3, 0.503 * h - 0.2] + list(coeffs)


def _image(n, w, h, seed):
    import cv2
    rng = np.random.default_rng(seed)
    return np.stack([cv2.GaussianBlur(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), (0, 0), 1.0)
                     for _ in range(n)])


def _kernel(imgs, model, prm, cam):
    w2, h2, pin = cam
    src = (colmap.MODEL_IDS[model][0], imgs.shape[2], imgs.shape[1], prm)
    return cio.undistort_u8(torch.from_numpy(imgs).to(DEV), src, (w2, h2, pin)).cpu().numpy()


@pytest.mark.parametrize("wh", [(161, 97), (1920, 1080)])
@pytest.mark.parametrize("model", list(COEFFS))
def test_kernel_matches_oracle(model, wh):
    w, h = wh
    prm = _params(model, w, h, COEFFS[model])
    cam = colmap.undistorted_camera(1, model, w, h, prm)
    imgs = _image(2, w, h, seed=w + len(model))
    got = _kernel(imgs, model, prm, cam)
    want = O.remap(imgs, model, prm, cam[2], cam[:2])
    assert got.shape == want.shape == (2, cam[1], cam[0], 3)
    for n in range(2):                                   # N = 1 gives each image's bytes
        assert np.array_equal(_kernel(imgs[n:n + 1], model, prm, cam)[0], got[n])
    diff = np.abs(got.astype(np.int16) - want)
    n_off = int((diff > 0).sum())
    print(f"{model} {w}x{h} -> {cam[0]}x{cam[1]}: {n_off} of {diff.size} bytes differ from the oracle")
    if model in O.FISHEYE:                               # atan may differ in the last bit
        assert diff.max() <= 1 and n_off < diff.size / 1e4
    else:
        assert n_off == 0
    assert (got[:, 2:-2, 2:-2] > 0).mean() > 0.9          # the map lands inside the source


@pytest.mark.parametrize("model", ["SIMPLE_RADIAL", "RADIAL", "OPENCV", "FULL_OPENCV"])
def test_zero_coefficients_are_the_identity(model):
    for w, h, cx, cy in ((161, 97, 80.3, 40.2), (1920, 1080, 955.1, 549.9), (64, 48, 31.0, 20.7)):
        focal = [0.8 * w] if model in O.SINGLE_FOCAL else [0.8 * w, 0.83 * w]
        prm = focal + [cx, cy] + [0.0] * (O.N_PARAMS[model] - len(focal) - 2)
        cam = colmap.undistorted_camera(1, model, w, h, prm)
        assert cam[:2] == (w, h)
        imgs = _image(2, w, h, seed=h)
        assert np.array_equal(_kernel(imgs, model, prm, cam), imgs), (model, w, h)


def _texture(x, y):
    """A smooth analytic texture of pinhole pixel coordinates, RGB, periods 40 to 64 px: at least
    16 px in the distorted image too, where the fisheye compresses its border up to 2.5 times."""
    a = np.sin(2 * np.pi * x / 48.0) * np.cos(2 * np.pi * y / 40.0)
    b = np.cos(2 * np.pi * (x + y) / 64.0)
    return np.stack([127.5 + 100 * a, 127.5 + 100 * b, 127.5 + 60 * (a * b)], -1)


@pytest.mark.parametrize("model", ["OPENCV", "OPENCV_FISHEYE", "RADIAL"])
def test_the_map_points_the_right_way(model):
    """The texture rendered through the distorted camera (each distorted pixel undistorted by
    the oracle's Newton inverse and looked up in the pinhole image plane), undistorted by the
    kernel, equals the texture rendered through the undistorted pinhole camera."""
    w, h = 320, 240
    prm = _params(model, w, h, COEFFS[model])
    w2, h2, pin = colmap.undistorted_camera(1, model, w, h, prm)
    fx, fy, cx2, cy2 = pin
    ys, xs = np.mgrid[:h, :w] + 0.5
    u, v, res = O.undistort(model, prm, xs.ravel(), ys.ravel())
    assert res.max() <= 1e-9
    dist = _texture((fx * u + cx2).reshape(h, w), (fy * v + cy2).reshape(h, w))
    dist = np.clip(np.floor(dist + 0.5), 0, 255).astype(np.uint8)
    got = _kernel(dist[None], model, prm, (w2, h2, pin))[0].astype(np.float64)
    ys2, xs2 = np.mgrid[:h2, :w2] + 0.5
    want = _texture(xs2, ys2)
    _, _, ok = O.source_map(model, prm, pin, (w2, h2), (w, h))
    inner = np.zeros_like(ok)
    inner[2:-2, 2:-2] = True
    from scipy.ndimage import binary_erosion
    keep = binary_erosion(ok, iterations=2) & inner
    assert keep.mean() > 0.5
    d = np.abs(got - want)[keep]
    print(f"{model}: mean |diff| {d.mean():.3f}, max {d.max():.1f} over {keep.sum()} pixels")
    assert d.mean() < 1.0 and d.max() <= 8


def _model():
    from casmvsnet_pl_b200 import ABN, synth
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN)
    synth.randomize_model_(model, 0)
    return model.eval().cuda()


DISTORTION = {1: ("OPENCV", [-0.12, 0.03, 1e-3, -5e-4]), 2: ("SIMPLE_RADIAL", [-0.09])}


def _run(net, root, out, **kw):
    scan = ep.ColmapScan(str(root), img_wh=(128, 96), n_views=3, **kw)
    ep.run_scan(net, scan, conf=0.0, min_geo_consistent=0, depth_dir=str(out / "depth"),
                ply_path=str(out / "s.ply"))
    d = out / "depth" / scan.scan
    return {f: (d / f).read_bytes() for f in sorted(os.listdir(d))}, (out / "s.ply").read_bytes()


def test_distorted_mapper_project_equals_the_pinhole_route(tmp_path):
    """A distorted capture in the mapper layout with its images elsewhere (--image_dir), against
    a pinhole workspace the test writes: the same views undistorted by the kernel, as PNG, and
    the model with the undistorted PINHOLE cameras."""
    cap, photos = tmp_path / "d" / "scene", tmp_path / "photos"
    model = synth_scenes.make_colmap(str(cap), n_views=6, image_wh=(150, 100), n_points=2000,
                                     seed=8, layout="mapper", image_ext="png",
                                     image_dir=str(photos), distortion=DISTORTION)
    from PIL import Image
    pin = tmp_path / "p" / "scene"
    os.makedirs(pin / "images")
    cams = {}
    for cid, (name, w, h, prm) in model.cameras.items():
        w2, h2, k = colmap.undistorted_camera(cid, name, w, h, prm)
        cams[cid] = ("PINHOLE", w2, h2, k)
        for q, t, c, img_name in model.images.values():
            if c == cid:
                img = np.asarray(Image.open(photos / img_name).convert("RGB"))
                und = _kernel(img[None].copy(), name, prm, (w2, h2, k))[0]
                Image.fromarray(und).save(pin / "images" / img_name)
    colmap.write_model(str(pin / "sparse"), colmap.ColmapModel(
        cams, model.images, model.point_ids, model.xyz, model.track_ptr, model.track_img), "bin")

    net = _model()
    dp, dply = _run(net, cap, tmp_path / "d_out", image_dir=str(photos))
    pp, pply = _run(net, pin, tmp_path / "p_out")
    assert dp.keys() == pp.keys() and len(dp) == 12
    for f in dp:
        assert dp[f] == pp[f], f
    assert dply == pply and len(dply) > 0

    out = tmp_path / "cli"
    ep.main(["--dataset_name", "colmap", "--root_dir", str(cap), "--image_dir", str(photos),
             "--out", str(out), "--img_wh", "128", "96", "--n_views", "3", "--conf", "0",
             "--min_geo_consistent", "0"])
    assert os.path.getsize(out / "points" / "scene.ply") > 0
    sc = colmap.load_scene(str(cap))
    assert sc.distorted.all()
    for v in range(len(sc)):
        K, E, _ = cio.read_cam_file(str(out / "scene" / "cams" / f"{v:08d}_cam.txt"))
        cid = next(c for _, _, c, n in model.images.values() if n == sc.names[v])
        name, w, h, prm = model.cameras[cid]
        w2, h2, k = colmap.undistorted_camera(cid, name, w, h, prm)
        assert np.array_equal(K, np.array([[k[0], 0, k[2]], [0, k[1], k[3]], [0, 0, 1]], np.float32))
        assert tuple(sc.wh[v]) == (w2, h2) and (w2, h2) != (w, h)


def test_image_of_the_wrong_size_is_refused_by_name(tmp_path):
    from PIL import Image
    root = tmp_path / "cap"
    model = synth_scenes.make_colmap(str(root), n_views=4, image_wh=(64, 48), n_points=300, seed=9,
                                     distortion=DISTORTION)
    name = sorted(im[3] for im in model.images.values())[2]
    Image.new("RGB", (70, 48)).save(root / "images" / name, quality=92)
    scan = ep.ColmapScan(str(root), img_wh=(64, 32), n_views=2)
    with pytest.raises(ValueError, match=f"{name}: the image is 70x48"):
        scan.fusion_images([0], DEV)


def test_host_images_with_a_distorted_camera_is_refused(tmp_path):
    root = tmp_path / "cap"
    synth_scenes.make_colmap(str(root), n_views=4, image_wh=(64, 48), n_points=300, seed=9,
                             distortion={2: ("SIMPLE_RADIAL", [-0.05])})
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match="host_images=True"):
        ep.ColmapScan(str(root), img_wh=(64, 32), n_views=2, host_images=True)
    assert _lib.launch_count() == n0
