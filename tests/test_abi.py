"""The C-ABI library loads and exports every symbol include/casmvs.h declares
(no compute calls: there is no GPU in the CPU test tier)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "casmvs.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(casmvs_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_expected_surface():
    syms = _declared_symbols()
    for must in ("casmvs_warp_cost_fwd", "casmvs_conv3d_fwd", "casmvs_costreg_fwd",
                 "casmvs_regress_fwd", "casmvs_depth_hypotheses_fwd", "casmvs_homo_warp_fwd",
                 "casmvs_device_check", "casmvs_last_error"):
        assert must in syms


def test_library_exports_every_declared_symbol():
    from casmvsnet_pl_b200 import _lib
    assert os.path.isfile(_lib.LIB_PATH), "build the extension first (__graft_entry__.build())"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in _declared_symbols():
        assert hasattr(lib, s), f"libcasmvs.so lacks {s}"


def test_binding_covers_header():
    from casmvsnet_pl_b200 import _lib
    assert sorted(_lib.SIGNATURES) == _declared_symbols()
    lib = _lib.load()
    assert lib.casmvs_version() == 100


def test_host_side_queries_without_gpu():
    from casmvsnet_pl_b200 import _lib, ops
    lib = _lib.load()
    assert lib.casmvs_packed_conv3d_weight_floats(32, 8) == 27 * 32 * 8
    assert lib.casmvs_warp_cost_workspace_bytes(_lib.NHWC, 1, 3, 32, 128, 160) == 0
    assert lib.casmvs_warp_cost_workspace_bytes(_lib.NCHW, 1, 3, 32, 128, 160) == 3 * 32 * 128 * 160 * 4
    total = lib.casmvs_costreg_param_floats(32)
    last = ops.costreg_layer_info(32, 10)
    assert last["cin"] == 8 and last["cout"] == 1 and last["shift_off"] + 1 == total
    first = ops.costreg_layer_info(32, 0)
    assert first["w_off"] == 0 and first["cin"] == 32 and first["cout"] == 8
    up = ops.costreg_layer_info(32, 7)
    assert up["kind"] == _lib.CONV_TRANSPOSE and (up["cin"], up["cout"]) == (64, 32)


def test_tensor_core_coverage_query_without_gpu():
    """ops.conv3d_tensor_core: every CostRegNet forward layer and the training adjoints that have
    a wgmma kernel say True; the adjoints that fall back (prob: 4 -> 8 after padding, the middle
    level's conv0: 8 -> 16), stride 2 with a skip, and Cin % 8 != 0 say False."""
    from casmvsnet_pl_b200 import ops
    C, T = ops.CONV, ops.CONV_TRANSPOSE
    for cin in (8, 16, 32):
        assert ops.conv3d_tensor_core(cin, 8, C, 1)
    for args in ((8, 16, C, 2), (16, 16, C, 1), (16, 32, C, 2), (32, 32, C, 1), (32, 64, C, 2),
                 (64, 64, C, 1), (64, 32, T, 2), (32, 16, T, 2), (16, 8, T, 2), (8, 1, C, 1),
                 (16, 8, C, 1), (32, 16, C, 1), (8, 32, C, 1)):
        assert ops.conv3d_tensor_core(*args), args
    for args in ((4, 8, C, 1), (8, 16, C, 1), (12, 8, C, 1), (16, 8, C, 2)):
        assert not ops.conv3d_tensor_core(*args), args
    assert not ops.conv3d_tensor_core(8, 16, C, 2, skip=True)
    assert ops.conv3d_tensor_core(64, 32, T, 2, skip=True)


def test_errors_are_reported_not_thrown():
    """bad arguments -> negative status + message (no GPU needed: validation is first)."""
    from casmvsnet_pl_b200 import _lib
    lib = _lib.load()
    rc = lib.casmvs_warp_cost_fwd(None, 1, None, None, None, 1, 1, 3, 8, 8, 16, 16, 1, None, 0, None)
    assert rc < 0 and b"null" in lib.casmvs_last_error()
    one = ctypes.c_void_p(16)
    rc = lib.casmvs_warp_cost_fwd(one, 1, one, one, one, 1, 1, 3, 12, 8, 16, 16, 1, None, 0, None)
    assert rc < 0 and b"multiple of 8" in lib.casmvs_last_error()
    rc = lib.casmvs_costreg_fwd(one, one, one, 1, 8, 12, 16, 16, 0, one, 1 << 40, None)
    assert rc < 0 and b"divisible by 8" in lib.casmvs_last_error()
    with pytest.raises(_lib.CasMVSError):
        _lib.check(rc, "costreg")


def test_costreg_blocked_coverage_is_pinned():
    """Every CostRegNet layer has a tensor-core kernel exactly for TF32 and Cin in {8, 16, 32}
    (conv1 .. prob always, conv0 for those input widths)."""
    from casmvsnet_pl_b200 import _lib
    lib = _lib.load()
    for cin in range(4, 65, 4):
        for prec in (_lib.FP32, _lib.TF32):
            want = int(prec == _lib.TF32 and cin in (8, 16, 32))
            assert lib.casmvs_costreg_blocked_supported(cin, prec) == want, (cin, prec)


def test_ladder_coverage_is_pinned():
    """The staged K1 kernel, the only one that takes a hypothesis ladder, covers one or two
    source views, C in {8, 16, 32}, variance or 8-group correlation."""
    from casmvsnet_pl_b200 import ops
    for V in range(2, 9):
        for C in range(4, 65, 4):
            for G in (1, 2, 4, 8):
                want = V - 1 in (1, 2) and C in (8, 16, 32) and G in (1, 8)
                assert ops.ladder_supported(V, C, G) is want, (V, C, G)


def test_misaligned_pointers_are_rejected():
    """Entry points whose kernels use 16-byte vectors reject a misaligned pointer before any
    device work, naming it (the message tells a rejection apart from "no device")."""
    from casmvsnet_pl_b200 import _lib
    lib = _lib.load()
    ok, bad = ctypes.c_void_p(0x10000), ctypes.c_void_p(0x10004)
    odd = ctypes.c_void_p(0x10002)

    def rejected(rc, what):
        msg = lib.casmvs_last_error()
        assert rc < 0 and what in msg and b"aligned" in msg, (rc, msg)

    NHWC, NCHW, CONV, TF32 = _lib.NHWC, _lib.NCHW, _lib.CONV, _lib.TF32
    # casmvs_conv3d_fwd: x always, y and skip when Cout > 1
    rejected(lib.casmvs_conv3d_fwd(bad, ok, ok, ok, 0.01, None, ok, 1, 8, 8, 8, 16, 16, CONV, 1,
                                   TF32, None), b"x must be 16-byte")
    rejected(lib.casmvs_conv3d_fwd(ok, ok, ok, ok, 0.01, None, bad, 1, 8, 8, 8, 16, 16, CONV, 1,
                                   TF32, None), b"y must be 16-byte")
    rejected(lib.casmvs_conv3d_fwd(ok, ok, ok, ok, 0.01, bad, ok, 1, 8, 8, 8, 16, 16, CONV, 1,
                                   TF32, None), b"skip must be 16-byte")
    rc = lib.casmvs_conv3d_fwd(ok, ok, ok, ok, 1.0, bad, bad, 1, 8, 1, 8, 16, 16, 7, 1, TF32, None)
    assert rc < 0 and b"bad kind" in lib.casmvs_last_error()        # Cout == 1: float stores
    # casmvs_costreg_fwd: x, workspace, logits
    rejected(lib.casmvs_costreg_fwd(bad, ok, ok, 1, 8, 16, 16, 16, TF32, ok, 1 << 30, None),
             b"x must be 16-byte")
    rejected(lib.casmvs_costreg_fwd(ok, ok, ok, 1, 8, 16, 16, 16, TF32, bad, 1 << 30, None),
             b"workspace must be 16-byte")
    rejected(lib.casmvs_costreg_fwd(ok, ok, odd, 1, 8, 16, 16, 16, TF32, ok, 1 << 30, None),
             b"logits must be 4-byte")
    # casmvs_warp_cost_fwd: NHWC features, the workspace of NCHW ones, an NHWC cost volume
    rejected(lib.casmvs_warp_cost_fwd(bad, NHWC, ok, ok, ok, NHWC, 1, 3, 8, 8, 16, 16, 1, None, 0,
                                      None), b"feats must be 16-byte")
    rejected(lib.casmvs_warp_cost_fwd(ok, NCHW, ok, ok, ok, NHWC, 1, 3, 8, 8, 16, 16, 1, bad,
                                      1 << 30, None), b"workspace must be 16-byte")
    rejected(lib.casmvs_warp_cost_fwd(ok, NHWC, ok, ok, bad, NHWC | _lib.ROUND_TF32, 1, 3, 8, 8,
                                      16, 16, 1, None, 0, None), b"cost must be 16-byte")
    # casmvs_warp_cost_ladder_fwd: features and cost volume
    rejected(lib.casmvs_warp_cost_ladder_fwd(bad, ok, None, None, 500.0, None, 2.5, ok, 1, 1, 3,
                                             8, 8, 16, 16, 1, None), b"feats must be 16-byte")
    rejected(lib.casmvs_warp_cost_ladder_fwd(ok, ok, None, None, 500.0, None, 2.5, bad,
                                             1 | _lib.BLOCKED, 1, 3, 8, 8, 16, 16, 1, None),
             b"cost must be 16-byte")
    # casmvs_homo_warp_fwd: features, an NHWC output
    rejected(lib.casmvs_homo_warp_fwd(bad, NHWC, ok, ok, ok, NCHW, 1, 8, 8, 16, 16, None),
             b"src_feat must be 16-byte")
    rejected(lib.casmvs_homo_warp_fwd(ok, NHWC, ok, ok, bad, NHWC, 1, 8, 8, 16, 16, None),
             b"warped must be 16-byte")
    rejected(lib.casmvs_conv2d_5x5s2_fwd(bad, ok, ok, 0.01, ok, 1, 8, 16, 32, 32, 1, None),
             b"x must be 16-byte")


def _header_constants():
    src = open(os.path.join(ROOT, "include", "casmvs.h")).read()
    consts = {k: int(v) for k, v in re.findall(r"#define\s+(CASMVS_[A-Z0-9_]+)\s+(\d+)", src)}
    for body in re.findall(r"enum\s+\w+\s*\{(.*?)\}", src, flags=re.S):
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        consts.update({k: int(v) for k, v in re.findall(r"(CASMVS_[A-Z0-9_]+)\s*=\s*(\d+)", body)})
    return consts


def test_binding_constants_match_header():
    """The ctypes binding re-states the header's enums and flags: keep them in lock step."""
    from casmvsnet_pl_b200 import _lib
    c = _header_constants()
    assert (c["CASMVS_NCHW"], c["CASMVS_NHWC"]) == (_lib.NCHW, _lib.NHWC)
    assert (c["CASMVS_FP32"], c["CASMVS_TF32"]) == (_lib.FP32, _lib.TF32)
    assert "CASMVS_TF32X3" not in c and "tf32x3" not in _lib.PRECISIONS   # removed, not lying
    assert (c["CASMVS_CONV"], c["CASMVS_CONV_TRANSPOSE"], c["CASMVS_CONV_PLANAR"]) == \
        (_lib.CONV, _lib.CONV_TRANSPOSE, _lib.CONV_PLANAR)
    assert c["CASMVS_ROUND_TF32"] == _lib.ROUND_TF32
    assert c["CASMVS_KEEP_FP32_OUT"] == _lib.KEEP_FP32_OUT
    # flags must not collide with the enum values they are OR-ed into
    assert c["CASMVS_ROUND_TF32"] > max(c["CASMVS_NCHW"], c["CASMVS_NHWC"])
    assert c["CASMVS_KEEP_FP32_OUT"] > c["CASMVS_TF32"]


def test_new_entry_points_validate_arguments():
    """FeatureNet entry points: argument validation comes before any device work."""
    from casmvsnet_pl_b200 import _lib
    lib = _lib.load()
    one = ctypes.c_void_p(16)
    rc = lib.casmvs_conv3d_fwd(one, one, None, None, 1.0, None, one, 1, 8, 8, 4, 16, 16,
                               _lib.CONV_PLANAR, 2, _lib.TF32, None)
    assert rc < 0 and b"stride" in lib.casmvs_last_error()
    rc = lib.casmvs_conv3d_fwd(one, one, None, None, 1.0, None, one, 1, 8, 8, 4, 16, 16,
                               _lib.CONV, 1, _lib.TF32 | 512, None)
    assert rc < 0 and b"precision" in lib.casmvs_last_error()
    rc = lib.casmvs_conv3d_fwd(one, one, None, None, 1.0, None, one, 1, 8, 8, 4, 16, 16,
                               _lib.CONV, 1, 2, None)            # the removed TF32X3 value
    assert rc < 0 and b"precision" in lib.casmvs_last_error()
    assert lib.casmvs_release_weight_images(one, 64) == 0         # nothing cached: no-op
    assert lib.casmvs_fallback_count() == 0 and lib.casmvs_weight_cache_generation() == 0
    rc = lib.casmvs_fpn_merge_fwd(one, one, one, one, one, 1, 15, 16, 8, 0, None)
    assert rc < 0 and b"even" in lib.casmvs_last_error()
    rc = lib.casmvs_fpn_merge_fwd(None, one, one, one, one, 1, 16, 16, 6, 0, None)
    assert rc < 0 and b"multiple of 4" in lib.casmvs_last_error()
    rc = lib.casmvs_conv2d_5x5s2_fwd(one, one, one, 0.01, one, 1, 8, 8, 32, 32, 0, None)
    assert rc < 0 and b"8->16" in lib.casmvs_last_error()
    rc = lib.casmvs_conv2d_rgb8_fwd(None, one, one, 0.01, one, 1, 32, 32, 0, None)
    assert rc < 0 and b"null" in lib.casmvs_last_error()
    assert lib.casmvs_conv2d_rgb8_fwd(one, one, one, 0.01, one, 0, 32, 32, 0, None) == 0   # empty batch
