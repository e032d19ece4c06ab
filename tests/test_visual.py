"""The training panels without a GPU: oracle/visual_oracle.py against the original project's
outputs recorded in tests/golden/visual (oracle/make_golden_visual.py), the committed colour-map
header against cv2, and the C ABI of casmvs_visual_panels."""
import ctypes
import glob
import os

import numpy as np
import pytest

from oracle import visual_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "visual")
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "*.npz"))
               if not p.endswith("cast.npz"))


def _load(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def _to_tensor(u8_hwc):
    """ToTensor of a uint8 image, as the original's visualize_* return it."""
    return u8_hwc.transpose(2, 0, 1).astype(np.float32) / np.float32(255)


def test_cases_cover_the_issue():
    assert {"dtu_640x512", "blendedmvs_768x576", "nan_inf", "constant", "conf_levels",
            "image_range", "wide_negative", "no_positive"} <= set(CASES)
    assert _load("dtu_640x512")["panel"].shape == (512, 4 * 640, 3)
    assert _load("blendedmvs_768x576")["panel"].shape == (576, 4 * 768, 3)
    z = _load("no_positive")
    assert z["vis_depth_gt_raises"] and z["vis_depth_pred_raises"] and not z["vis_prob_raises"]


def test_cast_rule_matches_numpy():
    z = _load("cast")
    assert (np.abs(z["x"][np.isfinite(z["x"])]) > 2.0 ** 31).sum() > 100
    assert np.array_equal(O.np_u8(z["x"]), z["u8"])
    assert O.np_u8(np.float32(-212.7)) == 44 and O.np_u8(np.float32(-1e6)) == 192


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(name):
    z = _load(name)
    assert np.array_equal(O.unpreprocess(z["img"]), z["unpreprocessed"])
    assert np.array_equal(_to_tensor(O.visualize_depth(z["depth_gt"])), z["vis_depth_gt"])
    assert np.array_equal(_to_tensor(O.visualize_depth(O.masked(z["depth_pred"], z["mask"]))),
                          z["vis_depth_pred"])
    assert np.array_equal(_to_tensor(O.visualize_prob(O.masked(z["conf"], z["mask"]))),
                          z["vis_prob"])
    panel = O.training_panel(z["img"], z["depth_gt"], z["depth_pred"], z["conf"], z["mask"])
    assert panel.dtype == np.uint8 and np.array_equal(panel, z["panel"])


def test_panels_swap_red_and_blue():
    """JET's low end is dark blue in cv2 (BGR (128, 0, 0)); the original shows it dark red."""
    assert tuple(O.visualize_depth(np.zeros((1, 1), np.float32))[0, 0]) == (128, 0, 0)
    grey0 = _load("no_positive")["panel"][:, 64:128]
    assert (grey0 == np.array([128, 0, 0], np.uint8)).all()


def test_colormap_header_equals_cv2():
    from casmvsnet_pl_b200 import colormap_table
    luts = O.colormaps()
    for name, lut in colormap_table.tables().items():
        assert np.array_equal(luts[name], lut), name
    path = colormap_table.HEADER
    assert open(path).read() == colormap_table.header_text()


def test_abi_entry_validates_arguments():
    from casmvsnet_pl_b200 import _lib
    lib = _lib.load()
    one = ctypes.c_void_p(16)
    rc = lib.casmvs_visual_panels(one, one, one, one, one, 0, 8, one, one, None)
    assert rc < 0 and b"bad dims" in lib.casmvs_last_error()
    rc = lib.casmvs_visual_panels(None, None, None, None, None, 8, 8, one, one, None)
    assert rc < 0 and b"no panel" in lib.casmvs_last_error()
    rc = lib.casmvs_visual_panels(None, one, None, None, None, 8, 8, one, None, None)
    assert rc < 0 and b"null workspace" in lib.casmvs_last_error()
    rc = lib.casmvs_visual_panels(None, one, None, None, None, 8, 8, one, ctypes.c_void_p(20), None)
    assert rc < 0 and b"aligned" in lib.casmvs_last_error()
    assert lib.casmvs_version() == 100


def test_tensorboard_flag_is_opt_in():
    """Without --tensorboard the namespace is the one of a run before the flag existed."""
    from casmvsnet_pl_b200 import train
    assert not hasattr(train.build_parser().parse_args([]), "tensorboard")
    assert train.build_parser().parse_args(["--tensorboard"]).tensorboard is True


def test_workspace_constant_matches_header():
    from casmvsnet_pl_b200 import _lib
    src = open(os.path.join(os.path.dirname(GOLDEN), "..", "..", "include", "casmvs.h")).read()
    assert f"#define CASMVS_VISUAL_WORKSPACE_BYTES {_lib.VISUAL_WORKSPACE_BYTES}" in src
