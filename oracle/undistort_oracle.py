"""CPU oracle of the undistortion of distorted COLMAP views (casmvsnet_pl_b200/colmap.py and
csrc/undistort.cu): float64 numpy restatements of

  distort(model, params, u, v)     COLMAP's forward distortion (du, dv) of normalised points
  undistort(model, params, x, y)   its inverse for pixels, by Newton's method with a
                                   central-difference Jacobian, and the round-trip residual (px)
  undistorted_camera(model, w, h, params)
                                   the project's undistorted-camera rule (README, "Your own
                                   scene"): (W', H', fx, fy, cx', cy') or ValueError
  remap(images, model, params, dst, wh)
                                   the kernel's map and bilinear sampling, operation for
                                   operation in the same order, so that every perspective model
                                   gives the kernel's bytes (numpy rounds every operation and
                                   never fuses a * b + c)

Test infrastructure only; the package never imports it.  tests/test_undistort.py pins distort
against OpenCV's projectPoints / fisheye.projectPoints.
"""
import math

import numpy as np

PINHOLES = ("SIMPLE_PINHOLE", "PINHOLE")
PERSPECTIVE = ("SIMPLE_RADIAL", "RADIAL", "OPENCV", "FULL_OPENCV")
FISHEYE = ("SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE", "OPENCV_FISHEYE")
MODEL_IDS = {"SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2, "RADIAL": 3, "OPENCV": 4,
             "OPENCV_FISHEYE": 5, "FULL_OPENCV": 6, "SIMPLE_RADIAL_FISHEYE": 8, "RADIAL_FISHEYE": 9}
N_PARAMS = {"SIMPLE_PINHOLE": 3, "PINHOLE": 4, "SIMPLE_RADIAL": 4, "RADIAL": 5, "OPENCV": 8,
            "OPENCV_FISHEYE": 8, "FULL_OPENCV": 12, "SIMPLE_RADIAL_FISHEYE": 4, "RADIAL_FISHEYE": 5}
SINGLE_FOCAL = ("SIMPLE_PINHOLE", "SIMPLE_RADIAL", "RADIAL", "SIMPLE_RADIAL_FISHEYE",
                "RADIAL_FISHEYE")
MIN_SCALE, MAX_SCALE = 0.2, 2.0


def split(model, params):
    """COLMAP parameters -> (fx, fy, cx, cy, distortion coefficients in COLMAP's order)."""
    p = [float(x) for x in params]
    if model in SINGLE_FOCAL:
        return p[0], p[0], p[1], p[2], p[3:]
    return p[0], p[1], p[2], p[3], p[4:]


def distort(model, params, u, v):
    """(du, dv) of normalised points (u, v), float64 arrays."""
    k = split(model, params)[4] + [0.0] * 8
    u, v = np.asarray(u, np.float64), np.asarray(v, np.float64)
    if model in PINHOLES:
        return np.zeros_like(u), np.zeros_like(v)
    u2, v2, uv = u * u, v * v, u * v
    r2 = u2 + v2
    if model in FISHEYE:
        r = np.sqrt(r2)
        th = np.arctan(r)
        t2 = th * th
        if model == "SIMPLE_RADIAL_FISHEYE":
            thd = th * (1.0 + k[0] * t2)
        elif model == "RADIAL_FISHEYE":
            t4 = t2 * t2
            thd = th * ((1.0 + k[0] * t2) + k[1] * t4)
        else:
            t4 = t2 * t2
            t6, t8 = t4 * t2, t4 * t4
            thd = th * ((((1.0 + k[0] * t2) + k[1] * t4) + k[2] * t6) + k[3] * t8)
        rs = np.where(r > 0, r, 1.0)
        return np.where(r > 0, (u * thd) / rs - u, 0.0), np.where(r > 0, (v * thd) / rs - v, 0.0)
    r4 = r2 * r2
    if model == "SIMPLE_RADIAL":
        return u * (k[0] * r2), v * (k[0] * r2)
    if model == "RADIAL":
        rad = k[0] * r2 + k[1] * r4
        return u * rad, v * rad
    p1, p2 = k[2], k[3]
    if model == "OPENCV":
        rad = k[0] * r2 + k[1] * r4
        return ((u * rad + (2.0 * p1) * uv) + p2 * (r2 + 2.0 * u2),
                (v * rad + (2.0 * p2) * uv) + p1 * (r2 + 2.0 * v2))
    assert model == "FULL_OPENCV", model
    r6 = r4 * r2
    rad = (((1.0 + k[0] * r2) + k[1] * r4) + k[4] * r6) / (((1.0 + k[5] * r2) + k[6] * r4) + k[7] * r6)
    return (((u * rad + (2.0 * p1) * uv) + p2 * (r2 + 2.0 * u2)) - u,
            ((v * rad + (2.0 * p2) * uv) + p1 * (r2 + 2.0 * v2)) - v)


def project(model, params, u, v):
    """Pixel (x, y) of normalised points: x = fx (u + du) + cx, y = fy (v + dv) + cy."""
    fx, fy, cx, cy, _ = split(model, params)
    du, dv = distort(model, params, u, v)
    return fx * (u + du) + cx, fy * (v + dv) + cy


def undistort(model, params, x, y, iters=100):
    """Normalised (u, v) with project(u, v) = (x, y), by Newton's method from the distorted point,
    and the round-trip residual max(|dx|, |dy|) in pixels."""
    fx, fy, cx, cy, _ = split(model, params)
    ud = (np.asarray(x, np.float64) - cx) / fx
    vd = (np.asarray(y, np.float64) - cy) / fy
    u, v = ud.copy(), vd.copy()
    for _ in range(iters):
        du, dv = distort(model, params, u, v)
        eu, ev = u + du - ud, v + dv - vd
        hu, hv = 1e-6 * np.maximum(1.0, np.abs(u)), 1e-6 * np.maximum(1.0, np.abs(v))
        a, b = distort(model, params, u + hu, v), distort(model, params, u - hu, v)
        c, d = distort(model, params, u, v + hv), distort(model, params, u, v - hv)
        j11 = 1.0 + (a[0] - b[0]) / (2 * hu)
        j21 = (a[1] - b[1]) / (2 * hu)
        j12 = (c[0] - d[0]) / (2 * hv)
        j22 = 1.0 + (c[1] - d[1]) / (2 * hv)
        det = j11 * j22 - j12 * j21
        su, sv = (j22 * eu - j12 * ev) / det, (j11 * ev - j21 * eu) / det
        u, v = u - su, v - sv
        if np.all(np.abs(su) <= 1e-15 * np.maximum(1.0, np.abs(u))) and \
                np.all(np.abs(sv) <= 1e-15 * np.maximum(1.0, np.abs(v))):
            break
    px, py = project(model, params, u, v)
    return u, v, np.maximum(np.abs(px - x), np.abs(py - y))


def undistorted_camera(model, w, h, params, min_scale=MIN_SCALE, max_scale=MAX_SCALE):
    """The undistorted PINHOLE camera of a distorted one -> (W', H', fx, fy, cx', cy')."""
    fx, fy, cx, cy, _ = split(model, params)
    if not all(math.isfinite(float(p)) for p in params) or not (fx > 0 and fy > 0):
        raise ValueError("parameters are not finite or a focal length is not positive")
    if w < 2 or h < 2:
        raise ValueError("size below 2 x 2")
    if not (0.5 < cx < w - 0.5 and 0.5 < cy < h - 0.5):
        raise ValueError("principal point outside the pixel-centre box")
    xs, ys = np.arange(w) + 0.5, np.arange(h) + 0.5
    border = {"left": (np.full(h, 0.5), ys), "right": (np.full(h, w - 0.5), ys),
              "top": (xs, np.full(w, 0.5)), "bottom": (xs, np.full(w, h - 0.5))}
    X, Y = {}, {}
    for side, (bx, by) in border.items():
        u, v, res = undistort(model, params, bx, by)
        if not np.all(res <= 1e-9):
            raise ValueError(f"the {side} border does not converge")
        X[side], Y[side] = fx * u + cx, fy * v + cy
    ratios = [(cx - X["left"].max()) / (cx - 0.5), (X["right"].min() - cx) / (w - 0.5 - cx),
              (cy - Y["top"].max()) / (cy - 0.5), (Y["bottom"].min() - cy) / (h - 0.5 - cy)]
    if not all(r > 0 for r in ratios):
        raise ValueError("a scale ratio is not positive")
    sx = min(max(min(ratios[0], ratios[1]), min_scale), max_scale)
    sy = min(max(min(ratios[2], ratios[3]), min_scale), max_scale)
    W2, H2 = max(2, math.floor(sx * w + 0.5)), max(2, math.floor(sy * h + 0.5))
    return W2, H2, fx, fy, cx * (W2 / w), cy * (H2 / h)


def source_map(model, params, dst, wh, src_wh):
    """Per output pixel: (sx, sy) source coordinates (pixel centres at integers) and whether the
    pixel is inside the source (within 1e-6), before clamping."""
    fx, fy, cx, cy, _ = split(model, params)
    ofx, ofy, ocx, ocy = (float(x) for x in dst)
    OW, OH = wh
    W, H = src_wh
    ys, xs = np.mgrid[:OH, :OW].astype(np.float64)
    u = ((xs + 0.5) - ocx) / ofx
    v = ((ys + 0.5) - ocy) / ofy
    du, dv = distort(model, params, u, v)
    sx = (fx * (u + du) + cx) - 0.5
    sy = (fy * (v + dv) + cy) - 0.5
    ok = (sx >= -1e-6) & (sx <= float(W - 1) + 1e-6) & (sy >= -1e-6) & (sy <= float(H - 1) + 1e-6)
    return sx, sy, ok


def remap(images, model, params, dst, wh):
    """(N,H,W,3) uint8 -> (N,OH,OW,3) uint8: the kernel's bilinear sample of every image at the
    source point of each output pixel, 0 outside, rounded by floor(s + 0.5)."""
    images = np.asarray(images)
    _, H, W, _ = images.shape
    sx, sy, ok = source_map(model, params, dst, wh, (W, H))
    sx = np.clip(np.where(ok, sx, 0.0), 0.0, float(W - 1))
    sy = np.clip(np.where(ok, sy, 0.0), 0.0, float(H - 1))
    x0 = np.minimum(np.floor(sx), W - 2).astype(np.int64)
    y0 = np.minimum(np.floor(sy), H - 2).astype(np.int64)
    ax, ay = (sx - x0)[..., None], (sy - y0)[..., None]
    bx, by = 1.0 - ax, 1.0 - ay
    p = images.astype(np.float64)
    s = by * (bx * p[:, y0, x0] + ax * p[:, y0, x0 + 1]) \
        + ay * (bx * p[:, y0 + 1, x0] + ax * p[:, y0 + 1, x0 + 1])
    out = np.clip(np.floor(s + 0.5), 0, 255).astype(np.uint8)
    out[:, ~ok] = 0
    return out
