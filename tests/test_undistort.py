"""Distorted COLMAP cameras, CPU tier: the oracle's forward distortion against OpenCV, the Newton
inverse, the undistorted-camera rule and its refusals, reading the seven distorted models (both
formats, the mapper layout), and the argument checks of casmvs_undistort_u8_fwd."""
import ctypes

import numpy as np
import pytest

from casmvsnet_pl_b200 import colmap, synth_scenes
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import undistort_oracle as O

# realistic coefficients of each model on a 640x480 camera
CAMERAS = {
    "SIMPLE_RADIAL": [520.0, 321.3, 238.6, -0.12],
    "RADIAL": [520.0, 321.3, 238.6, -0.15, 0.04],
    "OPENCV": [515.0, 522.0, 318.2, 243.9, -0.21, 0.05, 1.2e-3, -8e-4],
    "FULL_OPENCV": [515.0, 522.0, 318.2, 243.9, 0.35, -0.1, 1.2e-3, -8e-4, 0.02, 0.55, -0.05, 0.01],
    "SIMPLE_RADIAL_FISHEYE": [300.0, 320.5, 240.5, 0.03],
    "RADIAL_FISHEYE": [300.0, 320.5, 240.5, 0.03, -0.01],
    "OPENCV_FISHEYE": [300.0, 305.0, 318.0, 241.0, 0.04, -0.012, 0.003, -0.0004],
}
PERSPECTIVE = ("SIMPLE_RADIAL", "RADIAL", "OPENCV", "FULL_OPENCV")


def _opencv_project(model, params, u, v):
    import cv2
    fx, fy, cx, cy, k = O.split(model, params)
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    pts = np.stack([u, v, np.ones_like(u)], 1)
    zero = np.zeros(3)
    if model in O.FISHEYE:
        D = np.array((k + [0.0] * 4)[:4])
        out, _ = cv2.fisheye.projectPoints(pts[None], zero, zero, K, D)
    else:
        if model == "SIMPLE_RADIAL":
            D = [k[0], 0, 0, 0, 0, 0, 0, 0]
        elif model == "RADIAL":
            D = [k[0], k[1], 0, 0, 0, 0, 0, 0]
        elif model == "OPENCV":
            D = k + [0, 0, 0, 0]
        else:
            D = k
        out, _ = cv2.projectPoints(pts, zero, zero, K, np.array(D, np.float64))
    out = out.reshape(-1, 2)
    return out[:, 0], out[:, 1]


@pytest.mark.parametrize("model", list(CAMERAS))
def test_forward_distortion_matches_opencv(model):
    rng = np.random.default_rng(0)
    lim = 1.2 if model in O.FISHEYE else 0.6
    u, v = rng.uniform(-lim, lim, 2000), rng.uniform(-lim, lim, 2000)
    prm = CAMERAS[model]
    x, y = O.project(model, prm, u, v)
    cx_, cy_ = _opencv_project(model, prm, u, v)
    scale = np.maximum(np.abs(x), np.abs(y))
    assert np.max(np.abs(x - cx_) / scale) < 1e-12 and np.max(np.abs(y - cy_) / scale) < 1e-12
    # the package's own restatement (used for the camera rule) agrees with the oracle
    fx, fy, cx, cy, k = colmap.split_params(model, prm)
    du, dv = colmap.distortion(model, k, u, v)
    px, py = fx * (u + du) + cx, fy * (v + dv) + cy
    assert np.max(np.abs(px - x) / scale) < 1e-12 and np.max(np.abs(py - y) / scale) < 1e-12


@pytest.mark.parametrize("model", list(CAMERAS))
def test_newton_inverse_round_trips_over_the_image(model):
    ys, xs = np.mgrid[:480, :640] + 0.5
    u, v, res = O.undistort(model, CAMERAS[model], xs.ravel(), ys.ravel())
    assert res.max() <= 1e-9, res.max()
    x, y = O.project(model, CAMERAS[model], u, v)
    assert np.abs(x - xs.ravel()).max() <= 1e-9 and np.abs(y - ys.ravel()).max() <= 1e-9


@pytest.mark.parametrize("model", PERSPECTIVE)
def test_zero_coefficients_give_back_the_source_camera(model):
    for w, h, cx, cy in ((161, 97, 80.3, 40.2), (1920, 1080, 955.1, 549.9), (64, 48, 31.0, 20.7)):
        fx, fy = 500.0, 510.0
        f = [fx] if model in O.SINGLE_FOCAL else [fx, fy]
        fy = fx if model in O.SINGLE_FOCAL else fy
        prm = f + [cx, cy] + [0.0] * (O.N_PARAMS[model] - len(f) - 2)
        assert O.undistorted_camera(model, w, h, prm) == (w, h, fx, fy, cx, cy)
        w2, h2, pin = colmap.undistorted_camera(1, model, w, h, prm)
        assert (w2, h2) == (w, h) and pin.tolist() == [fx, fy, cx, cy]


def test_barrel_grows_and_pincushion_shrinks_the_camera():
    for k, grows in ((-0.08, True), (0.08, False)):
        w2, h2, _ = colmap.undistorted_camera(1, "SIMPLE_RADIAL", 1920, 1080, [1600, 960.3, 540.7, k])
        assert (w2 > 1920 and h2 > 1080) if grows else (w2 < 1920 and h2 < 1080)


def test_worked_examples():
    cases = [("SIMPLE_RADIAL", [1600, 960.3, 540.7, -0.08], (1981, 1090)),
             ("SIMPLE_RADIAL", [1600, 960.3, 540.7, 0.08], (1854, 1043)),
             ("OPENCV_FISHEYE", [800, 800, 960, 540, 0.05, -0.01, 0.002, 0], (3480, 1246))]
    for model, prm, wh in cases:
        want = O.undistorted_camera(model, 1920, 1080, prm)
        assert want[:2] == wh
        w2, h2, pin = colmap.undistorted_camera(1, model, 1920, 1080, prm)
        assert (w2, h2) == wh
        assert np.allclose(pin, want[2:], rtol=1e-12, atol=0)
    assert O.undistorted_camera("OPENCV_FISHEYE", 1920, 1080, cases[2][1])[4] == 960 * (3480 / 1920)


def test_a_wide_fisheye_clips_at_two():
    w2, h2, pin = colmap.undistorted_camera(1, "SIMPLE_RADIAL_FISHEYE", 1920, 1080, [720, 960, 540, 0.0])
    assert w2 == 2 * 1920 and h2 < 2 * 1080
    assert O.undistorted_camera("SIMPLE_RADIAL_FISHEYE", 1920, 1080, [720, 960, 540, 0.0])[:2] == (w2, h2)


@pytest.mark.parametrize("model,w,h,prm,why", [
    ("SIMPLE_RADIAL_FISHEYE", 1920, 1080, [700, 960, 540, 0.0], "does not converge"),
    ("SIMPLE_RADIAL", 640, 480, [500, 0.3, 240, 0.1], "principal point"),
    ("SIMPLE_RADIAL", 640, 480, [500, 320, 479.7, 0.1], "principal point"),
    ("OPENCV", 640, 480, [500, 500, 5, 240, 0, 0, 0, -0.05], "ratio is not positive"),
    ("SIMPLE_RADIAL", 1, 480, [500, 0.3, 240, 0.1], "below 2 x 2"),
    ("SIMPLE_RADIAL", 640, 480, [500, 320, 240, np.nan], "not finite"),
    ("OPENCV", 640, 480, [500, np.inf, 320, 240, 0, 0, 0, 0], "not finite"),
    ("OPENCV", 640, 480, [500, -500, 320, 240, 0, 0, 0, 0], "focal length"),
])
def test_camera_refusals_name_the_camera(model, w, h, prm, why):
    with pytest.raises(ValueError, match=f"camera 7 .*{why}"):
        colmap.undistorted_camera(7, model, w, h, prm)
    with pytest.raises(ValueError):
        O.undistorted_camera(model, w, h, prm)


def _distortion(model):
    """A synthetic capture's cameras as `model`: camera 2 (SIMPLE_PINHOLE) always, camera 1
    (PINHOLE, fx != fy) too when the model has two focal lengths."""
    k = {"SIMPLE_RADIAL": [-0.1], "RADIAL": [-0.1, 0.02], "OPENCV": [-0.1, 0.02, 1e-3, -1e-3],
         "FULL_OPENCV": [-0.1, 0.02, 1e-3, -1e-3, 0.01, 0.05, -0.01, 0.002],
         "SIMPLE_RADIAL_FISHEYE": [0.02], "RADIAL_FISHEYE": [0.02, -0.005],
         "OPENCV_FISHEYE": [0.02, -0.005, 1e-3, -1e-4]}[model]
    d = {2: (model, k)}
    if model not in O.SINGLE_FOCAL:
        d[1] = (model, k)
    return d


@pytest.mark.parametrize("model", list(CAMERAS))
@pytest.mark.parametrize("fmt,layout", [("bin", "mapper"), ("txt", "mapper"), ("bin", "undistorted")])
def test_distorted_models_are_read(tmp_path, model, fmt, layout):
    m = synth_scenes.make_colmap(str(tmp_path), n_views=4, image_wh=(64, 48), n_points=200, seed=3,
                                 fmt=fmt, layout=layout, distortion=_distortion(model))
    sparse = colmap.find_sparse_dir(str(tmp_path))
    assert sparse.endswith("0") == (layout == "mapper")
    with pytest.raises(ValueError, match=f"{model}.*image_undistorter"):
        colmap.read_model(sparse)
    sc = colmap.load_scene(str(tmp_path))
    by_name = {im[3]: im[2] for im in m.images.values()}
    for v, name in enumerate(sc.names):
        cname, w, h, prm = m.cameras[by_name[name]]
        assert sc.src_cameras[v][0] == colmap.MODEL_IDS[cname][0]
        assert sc.src_cameras[v][1:3] == (w, h) and np.array_equal(sc.src_cameras[v][3], prm)
        assert sc.distorted[v] == (cname != "PINHOLE")
        if sc.distorted[v]:
            w2, h2, fx, fy, cx, cy = O.undistorted_camera(cname, w, h, prm)
            assert tuple(sc.wh[v]) == (w2, h2)
            assert np.allclose([sc.K[v, 0, 0], sc.K[v, 1, 1], sc.K[v, 0, 2], sc.K[v, 1, 2]],
                               [fx, fy, cx, cy], rtol=1e-12, atol=0)
        else:
            assert tuple(sc.wh[v]) == (w, h) and np.array_equal(sc.K[v], colmap.intrinsics(cname, prm))


@pytest.mark.parametrize("model", ["FOV", "THIN_PRISM_FISHEYE"])
def test_unsupported_models_are_refused_by_name(tmp_path, model):
    m = synth_scenes.colmap_model(n_views=4, n_points=100, seed=4)
    m.cameras[2] = (model, 200, 150, np.array([200.0, 100.0, 75.0] + [0.01] * (colmap.MODEL_IDS[model][1] - 3)))
    colmap.write_model(str(tmp_path), m, "bin")
    with pytest.raises(ValueError, match=f"camera 2 uses the {model} model, which is not supported"):
        colmap.read_model(str(tmp_path), distorted=True)
    with pytest.raises(ValueError, match=model):
        colmap.load_scene(str(tmp_path))


def test_a_refused_camera_is_named_when_read(tmp_path):
    m = synth_scenes.colmap_model(n_views=4, n_points=100, seed=4)
    m.cameras[2] = ("SIMPLE_RADIAL", 200, 150, np.array([200.0, 0.2, 75.0, 0.1]))
    colmap.write_model(str(tmp_path), m, "txt")
    with pytest.raises(ValueError, match="camera 2 .*principal point"):
        colmap.load_scene(str(tmp_path))


def test_defaults_leave_the_synthetic_capture_unchanged(tmp_path):
    a = synth_scenes.make_colmap(str(tmp_path / "a"), n_views=4, image_wh=(64, 48), n_points=200, seed=5)
    b = synth_scenes.colmap_model(n_views=4, image_wh=(64, 48), n_points=200, seed=5,
                                  distortion={2: ("SIMPLE_RADIAL", [0.01])})
    assert sorted(im[3] for im in a.images.values())[0] == "view_000.jpg"
    assert a.cameras[1][0] == "PINHOLE" and b.cameras[1][0] == "PINHOLE"
    assert b.cameras[2][0] == "SIMPLE_RADIAL" and b.cameras[2][3].tolist() == a.cameras[2][3].tolist() + [0.01]
    assert np.array_equal(a.track_img, b.track_img) and np.array_equal(a.xyz, b.xyz)
    with pytest.raises(ValueError, match="one focal length"):
        synth_scenes.colmap_model(n_views=4, n_points=100, seed=5, distortion=("SIMPLE_RADIAL", [0.01]))


def test_image_dir_applies_to_colmap_only(tmp_path):
    with pytest.raises(SystemExit, match="--image_dir"):
        ep.main(["--root_dir", str(tmp_path), "--dataset_name", "tanks", "--split", "intermediate",
                 "--image_dir", str(tmp_path)])
    assert ep.parse_args(["--root_dir", "r", "--dataset_name", "colmap"]).image_dir is None


def test_undistort_entry_validates_before_any_cuda_call():
    from casmvsnet_pl_b200 import _lib
    lib = _lib.load()
    one = ctypes.c_void_p(256)
    src = (ctypes.c_double * 12)(500, 500, 80, 60, *([0.0] * 8))
    dst = (ctypes.c_double * 4)(500, 500, 80, 60)
    for model in (7, 10, 11, -1):
        rc = lib.casmvs_undistort_u8_fwd(one, one, 1, 120, 160, 120, 160, model, src, dst, None)
        assert rc < 0 and b"unsupported camera model id" in lib.casmvs_last_error()
    for n, h, w, oh, ow in ((-1, 120, 160, 120, 160), (1, 1, 160, 120, 160), (1, 120, 1, 120, 160),
                            (1, 120, 160, 0, 160), (1, 120, 160, 120, -3)):
        rc = lib.casmvs_undistort_u8_fwd(one, one, n, h, w, oh, ow, 4, src, dst, None)
        assert rc < 0 and b"bad dims" in lib.casmvs_last_error()
    rc = lib.casmvs_undistort_u8_fwd(one, one, 1, 120, 160, 120, 160, 4, None, dst, None)
    assert rc < 0 and b"null parameter" in lib.casmvs_last_error()
    rc = lib.casmvs_undistort_u8_fwd(None, one, 1, 120, 160, 120, 160, 4, src, dst, None)
    assert rc < 0 and b"null pointer" in lib.casmvs_last_error()
    bad = (ctypes.c_double * 4)(500, 0, 80, 60)
    rc = lib.casmvs_undistort_u8_fwd(one, one, 1, 120, 160, 120, 160, 4, src, bad, None)
    assert rc < 0 and b"focal" in lib.casmvs_last_error()
    assert lib.casmvs_undistort_u8_fwd(None, None, 0, 120, 160, 120, 160, 4, src, dst, None) == 0
