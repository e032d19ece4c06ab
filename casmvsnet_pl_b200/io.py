"""Input pipeline and on-disk formats either side of the hot path (SURVEY.md §8 f-4).

Host-side Python like the reference's (it is data plumbing, not arithmetic on the path):

  read_pfm / save_pfm          reference datasets/utils.py:5-69 (PFM, bottom-up rows, scale sign
                               = endianness) -- byte-compatible both ways
  read_cam_file                reference datasets/dtu.py:77-90 (MVSNet cam.txt)
  read_pair_file               reference datasets/dtu.py:41-50 (pair.txt)
  pyramid_proj_mats            reference datasets/dtu.py:52-75 (K[R|t] per level, fine -> coarse,
                               intrinsics doubled per finer level, optional test-mode rescale)
  relative_proj_mats           reference datasets/dtu.py:181-186 (src_proj @ inv(ref_proj), rows 0..2)
  normalize_images             reference datasets/dtu.py:130-137 (ToTensor + ImageNet Normalize):
                               uint8 HWC images are uploaded AS BYTES (4x less H2D traffic than
                               fp32) and converted + normalised + re-laid-out to planar fp32 on the
                               GPU by casmvs_normalize_u8_fwd
  read_ply                     PLY vertices (binary little-endian or ASCII, scalar properties): reads
                               fusion.write_ply output and the DTU ground-truth STL clouds
  DepthWriter / infer_views    reference eval.py:213-229 (the per-view inference loop): views are
                               streamed through PipelinedCascade (H2D, forward and D2H of
                               neighbouring views overlap), NaNs scrubbed, depth_XXXX.pfm and
                               proba_XXXX.pfm written in the reference's layout
"""
from __future__ import annotations

import os
import re
import sys

import numpy as np
import torch

IMAGENET_MEAN = (0.485, 0.456, 0.406)      # datasets/dtu.py:133-134
IMAGENET_STD = (0.229, 0.224, 0.225)


# ------------------------------------------------------------------------------ PFM
def read_pfm(filename):
    """-> (data float32 (H,W) or (H,W,3), scale).  datasets/utils.py:5-39."""
    with open(filename, "rb") as f:
        header = f.readline().decode("utf-8").rstrip()
        if header == "PF":
            color = True
        elif header == "Pf":
            color = False
        else:
            raise ValueError("Not a PFM file.")
        m = re.match(r"^(\d+)\s(\d+)\s$", f.readline().decode("utf-8"))
        if not m:
            raise ValueError("Malformed PFM header.")
        width, height = map(int, m.groups())
        scale = float(f.readline().rstrip())
        endian = "<" if scale < 0 else ">"        # negative scale = little-endian
        scale = abs(scale)
        data = np.frombuffer(f.read(), dtype=endian + "f4")
    shape = (height, width, 3) if color else (height, width)
    if data.size != int(np.prod(shape)):
        raise ValueError(f"PFM payload has {data.size} floats, header says {shape}")
    return np.flipud(data.reshape(shape)), scale


def save_pfm(filename, image, scale=1):
    """datasets/utils.py:42-69: float32 only, rows bottom-up, scale sign = byte order."""
    image = np.asarray(image)
    if image.dtype.name != "float32":
        raise TypeError("Image dtype must be float32.")
    if image.ndim == 3 and image.shape[2] == 3:
        color = True
    elif image.ndim == 2 or (image.ndim == 3 and image.shape[2] == 1):
        color = False
    else:
        raise ValueError("Image must have H x W x 3, H x W x 1 or H x W dimensions.")
    endian = image.dtype.byteorder
    if endian == "<" or (endian == "=" and sys.byteorder == "little"):
        scale = -scale
    with open(filename, "wb") as f:
        f.write(b"PF\n" if color else b"Pf\n")
        f.write(f"{image.shape[1]} {image.shape[0]}\n".encode("utf-8"))
        f.write(("%f\n" % scale).encode("utf-8"))
        np.ascontiguousarray(np.flipud(image)).tofile(f)


# ------------------------------------------------------------------------------ PLY
_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2",
              "int16": "i2", "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4",
              "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8",
              "float64": "f8"}


def read_ply(filename):
    """-> numpy structured array of the vertex element, one field per property.

    Reads `format binary_little_endian 1.0` and `format ascii 1.0` files whose vertex element is
    the first element and has scalar properties only; elements after it (faces, ...) are ignored.
    Anything else (big-endian, list properties on vertices, a missing vertex element) raises
    ValueError."""
    with open(filename, "rb") as f:
        if f.readline().rstrip(b"\r\n") != b"ply":
            raise ValueError(f"{filename}: not a PLY file")
        fmt, elements = None, []
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{filename}: PLY header has no end_header")
            tok = line.decode("ascii", "replace").split()
            if not tok or tok[0] in ("comment", "obj_info"):
                continue
            if tok[0] == "end_header":
                break
            if tok[0] == "format":
                fmt = tok[1] if len(tok) == 3 and tok[2] == "1.0" else None
                if fmt not in ("binary_little_endian", "ascii"):
                    raise ValueError(f"{filename}: unsupported PLY format {' '.join(tok[1:])}")
            elif tok[0] == "element" and len(tok) == 3:
                elements.append((tok[1], int(tok[2]), []))
            elif tok[0] == "property" and elements:
                if tok[1] == "list" or len(tok) != 3 or tok[1] not in _PLY_TYPES:
                    elements[-1][2].append(None)            # unsupported; fatal only on vertices
                else:
                    elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]]))
            else:
                raise ValueError(f"{filename}: malformed PLY header line {line!r}")
        if fmt is None:
            raise ValueError(f"{filename}: PLY header has no format line")
        if not elements or elements[0][0] != "vertex":
            raise ValueError(f"{filename}: the first PLY element must be 'vertex'")
        _, n, props = elements[0]
        if not props or any(p is None for p in props):
            raise ValueError(f"{filename}: vertex properties must be scalars")
        if fmt == "binary_little_endian":
            dtype = np.dtype([(name, "<" + t) for name, t in props])
            data = np.frombuffer(f.read(n * dtype.itemsize), dtype=dtype)
            if len(data) != n:
                raise ValueError(f"{filename}: {len(data)} vertices, header says {n}")
            return data.copy()
        dtype = np.dtype([(name, t) for name, t in props])
        rows = [f.readline().split() for _ in range(n)]
    if any(len(r) != len(props) for r in rows):
        raise ValueError(f"{filename}: ASCII vertex rows must hold {len(props)} values")
    out = np.empty(n, dtype=dtype)
    cols = np.array(rows, dtype=object).reshape(n, len(props))
    for j, (name, t) in enumerate(props):
        out[name] = cols[:, j].astype(np.float64 if t[0] == "f" else np.int64).astype(t) if n else []
    return out


# ------------------------------------------------------------------------------ cameras
def read_cam_file(filename):
    """MVSNet cam.txt -> (intrinsics (3,3) f32, extrinsics (4,4) f32, depth_min float).
    datasets/dtu.py:77-90: extrinsics on lines [1,5), intrinsics on lines [7,10), depth_min first
    token of line 11."""
    with open(filename) as f:
        lines = [line.rstrip() for line in f.readlines()]
    extrinsics = np.array(" ".join(lines[1:5]).split(), dtype=np.float32).reshape(4, 4)
    intrinsics = np.array(" ".join(lines[7:10]).split(), dtype=np.float32).reshape(3, 3)
    depth_min = float(lines[11].split()[0])
    return intrinsics, extrinsics, depth_min


def read_pair_file(filename):
    """pair.txt -> [(ref_view, [src views by score])].  datasets/dtu.py:41-50 (ids are every
    second token of the score line)."""
    out = []
    with open(filename) as f:
        n = int(f.readline())
        for _ in range(n):
            ref = int(f.readline().rstrip())
            src = [int(x) for x in f.readline().rstrip().split()[1::2]]
            out.append((ref, src))
    return out


def pyramid_proj_mats(intrinsics, extrinsics, levels=3, img_wh=None, full_wh=(1600, 1200)):
    """(levels,4,4) float32 world->pixel matrices, level 0 = finest.  datasets/dtu.py:52-75:
    `intrinsics` are those of the COARSEST level (cam files hold quarter-resolution values);
    in test mode (img_wh given) they are first rescaled by img_wh / full_wh / 4.  Arithmetic in
    float32 numpy like the reference (np.eye is float64, the product is float32 @ float32 placed
    into it, then cast by torch.FloatTensor)."""
    K = np.array(intrinsics, dtype=np.float32, copy=True)
    E = np.asarray(extrinsics, dtype=np.float32)
    if img_wh is not None:
        K[0] *= img_wh[0] / full_wh[0] / 4
        K[1] *= img_wh[1] / full_wh[1] / 4
    mats = []
    for _ in range(levels):
        P = np.eye(4)
        P[:3, :4] = K @ E[:3, :4]
        K[:2] *= 2                                   # 1/4 -> 1/2 -> 1
        mats.append(torch.FloatTensor(P))
    return torch.stack(mats[::-1])


def relative_proj_mats(proj_mats_by_view, view_ids):
    """view_ids = [ref, src...] -> (V-1, levels, 3, 4): src_proj @ inv(ref_proj), rows 0..2,
    what CascadeMVSNet.forward takes (datasets/dtu.py:176-186)."""
    ref_inv = torch.inverse(proj_mats_by_view[view_ids[0]])
    return torch.stack([proj_mats_by_view[v] @ ref_inv for v in view_ids[1:]])[:, :, :3]


# ------------------------------------------------------------------------------ images
def normalize_images(images_u8, device=None, out=None):
    """uint8 (N,H,W,3) RGB images -> float32 (N,3,H,W), (x/255 - mean)/std per channel
    (ToTensor + Normalize, datasets/dtu.py:130-137) on the GPU.  `images_u8` may be a pinned
    host tensor (uploaded as bytes: 4x less H2D traffic than normalised floats) or already on
    the device.  Matches the torchvision arithmetic: x.float().div(255).sub(mean).div(std)."""
    import ctypes

    from . import _lib
    t = images_u8 if torch.is_tensor(images_u8) else torch.from_numpy(np.ascontiguousarray(images_u8))
    if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[-1] != 3:
        raise _lib.CasMVSError("normalize_images expects uint8 (N,H,W,3)")
    if not t.is_cuda:
        if device is None:
            raise _lib.CasMVSError("normalize_images: give a CUDA device for host input (no CPU path)")
        t = t.to(device, non_blocking=True)
    t = t.contiguous()
    N, H, W, _ = t.shape
    if out is None:
        out = torch.empty(N, 3, H, W, device=t.device, dtype=torch.float32)
    mean = (ctypes.c_float * 3)(*IMAGENET_MEAN)
    std = (ctypes.c_float * 3)(*IMAGENET_STD)
    with torch.cuda.device(t.device):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(_lib.load().casmvs_normalize_u8_fwd(
            ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(out.data_ptr()), N, H, W, mean, std, st),
            "normalize_u8")
    return out


_PIL_PRECISION_BITS = 22        # Pillow Resample.c PRECISION_BITS (8-bit images)
_CV_COEF_SCALE = 2048           # OpenCV INTER_RESIZE_COEF_SCALE (1 << 11)


def pil_bilinear_coeffs(in_size, out_size):
    """Pillow's BILINEAR coefficients along one axis of `in_size` -> `out_size` pixels:
    bounds (out,2) int32 = (first tap, taps), coef (out,ksize) int32.  In double: support =
    max(scale, 1), triangle filter, normalised by the sequential sum; then rounded half away from
    zero to 22 fractional bits (Resample.c precompute_coeffs / normalize_coeffs_8bpc)."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    ss = 1.0 / filterscale
    ksize = int(np.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    coef = np.zeros((out_size, ksize), np.int32)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - xmin
        w = [max(0.0, 1.0 - abs((x + xmin - center + 0.5) * ss)) for x in range(n)]
        total = 0.0
        for v in w:
            total += v
        for x, v in enumerate(w):
            v = v / total if total != 0.0 else v
            coef[xx, x] = int(0.5 + v * (1 << _PIL_PRECISION_BITS)) if v >= 0 else \
                int(-0.5 + v * (1 << _PIL_PRECISION_BITS))
        bounds[xx] = (xmin, n)
    return bounds, coef


def cv2_linear_table(in_size, out_size, clamp):
    """OpenCV INTER_LINEAR taps along one axis -> (out,4) int32 (i0, i1, w0, w1).  Source
    position fx = (float)((d + 0.5) * (1 / (out/in)) - 0.5), split into floor and fraction in
    float32, weights saturate_cast<short>((1 - f, f) * 2048) (round half even).  Along x
    (`clamp`) positions left of 0 or at/right of the last pixel take that pixel alone; along y
    the weights are kept and only the row indices are clipped (resize.cpp)."""
    scale = 1.0 / (out_size / in_size)
    f = ((np.arange(out_size, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp:
        lo, hi = s < 0, s >= in_size - 1
        f[lo | hi] = 0
        s[lo], s[hi] = 0, in_size - 1
    w1 = np.rint(f * np.float32(_CV_COEF_SCALE)).astype(np.int64)
    w0 = np.rint((np.float32(1) - f) * np.float32(_CV_COEF_SCALE)).astype(np.int64)
    return np.stack([np.clip(s, 0, in_size - 1), np.clip(s + 1, 0, in_size - 1), w0, w1],
                    1).astype(np.int32)


_TABLES = {}


def _device_tables(kind, hw, ohw, device):
    key = (kind, hw, ohw, str(device))
    if key not in _TABLES:
        (H, W), (OH, OW) = hw, ohw
        if kind == "pil":
            xb, xc = pil_bilinear_coeffs(W, OW)
            yb, yc = pil_bilinear_coeffs(H, OH)
            t = [torch.from_numpy(a).to(device) for a in (xb, xc, yb, yc)]
        else:
            t = [torch.from_numpy(cv2_linear_table(W, OW, True)).to(device),
                 torch.from_numpy(cv2_linear_table(H, OH, False)).to(device)]
        _TABLES[key] = t
    return _TABLES[key]


def _check_u8_images(images, what):
    from . import _lib
    if not torch.is_tensor(images) or not images.is_cuda or images.dtype != torch.uint8 \
            or images.dim() != 4 or images.shape[-1] != 3:
        raise _lib.CasMVSError(f"{what} expects a uint8 (N,H,W,3) CUDA tensor")
    return images.contiguous()


def resize_u8_pil(images, wh, out=None):
    """Pillow Image.resize(wh, Image.BILINEAR) of uint8 (N,H,W,3) CUDA images ->
    (N,h,w,3) uint8, byte-identical (casmvs_resize_u8_pil_fwd)."""
    import ctypes

    from . import _lib
    t = _check_u8_images(images, "resize_u8_pil")
    N, H, W, _ = t.shape
    OW, OH = int(wh[0]), int(wh[1])
    if OW <= 0 or OH <= 0:
        raise _lib.CasMVSError(f"resize_u8_pil: bad size {tuple(wh)}")
    if out is None:
        out = torch.empty(N, OH, OW, 3, device=t.device, dtype=torch.uint8)
    xb, xc, yb, yc = _device_tables("pil", (H, W), (OH, OW), t.device)
    tmp = torch.empty(N, H, OW, 3, device=t.device, dtype=torch.uint8) \
        if OW != W and OH != H else None
    p = lambda x: ctypes.c_void_p(x.data_ptr() if x is not None else 0)   # noqa: E731
    with torch.cuda.device(t.device):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(_lib.load().casmvs_resize_u8_pil_fwd(
            p(t), p(out), p(tmp), N, H, W, OH, OW, p(xb), p(xc), xc.shape[1], p(yb), p(yc),
            yc.shape[1], st), "resize_u8_pil")
    return out


def resize_u8_linear(images, wh, out=None):
    """cv2.resize(img, wh, interpolation=cv2.INTER_LINEAR) of uint8 (N,H,W,3) CUDA images ->
    (N,h,w,3) uint8, byte-identical (casmvs_resize_u8_linear_fwd)."""
    import ctypes

    from . import _lib
    t = _check_u8_images(images, "resize_u8_linear")
    N, H, W, _ = t.shape
    OW, OH = int(wh[0]), int(wh[1])
    if OW <= 0 or OH <= 0:
        raise _lib.CasMVSError(f"resize_u8_linear: bad size {tuple(wh)}")
    if out is None:
        out = torch.empty(N, OH, OW, 3, device=t.device, dtype=torch.uint8)
    xt, yt = _device_tables("cv2", (H, W), (OH, OW), t.device)
    with torch.cuda.device(t.device):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(_lib.load().casmvs_resize_u8_linear_fwd(
            ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(out.data_ptr()), N, H, W, OH, OW,
            ctypes.c_void_p(xt.data_ptr()), ctypes.c_void_p(yt.data_ptr()), st),
            "resize_u8_linear")
    return out


def save_visual(depth_dir, scan, vid, depth, proba, conf):
    """eval.py:230-239: JET-coloured depth (min over positive depths .. max, to uint8) and the
    confidence mask proba > conf as JPEGs next to the PFMs."""
    import cv2
    d = os.path.join(depth_dir, scan)
    os.makedirs(d, exist_ok=True)
    mi = np.min(depth[depth > 0])
    ma = np.max(depth)
    depth = (255 * ((depth - mi) / (ma - mi + 1e-8))).astype(np.uint8)
    cv2.imwrite(os.path.join(d, f"depth_visual_{vid:04d}.jpg"), cv2.applyColorMap(depth, cv2.COLORMAP_JET))
    cv2.imwrite(os.path.join(d, f"proba_visual_{vid:04d}.jpg"), (255 * (proba > conf)).astype(np.uint8))


# ------------------------------------------------------------------------------ eval loop
def scrub(x):
    """np.nan_to_num of eval.py:225-227 (NaN -> 0; +-inf -> largest finite)."""
    return np.nan_to_num(x)


class DepthWriter:
    """results/<dataset>/depth/<scan>/depth_XXXX.pfm + proba_XXXX.pfm (eval.py:228-229)."""

    def __init__(self, depth_dir):
        self.depth_dir = depth_dir

    def __call__(self, scan, vid, depth, proba):
        d = os.path.join(self.depth_dir, scan)
        os.makedirs(d, exist_ok=True)
        save_pfm(os.path.join(d, f"depth_{vid:04d}.pfm"), scrub(np.asarray(depth, dtype=np.float32)))
        save_pfm(os.path.join(d, f"proba_{vid:04d}.pfm"), scrub(np.asarray(proba, dtype=np.float32)))


def infer_views(model, views, init_depth_min, depth_interval, sink, device="cuda:0"):
    """The inference loop of eval.py:213-229 for views of one shape, streamed: `views` yields
    (key, imgs (V,3,H,W) float32 host tensor, proj_mats (V-1,levels,3,4) host tensor); for each,
    `sink(key, depth_0 (H,W) ndarray, confidence_2 (H/4,W/4) ndarray)` is called in order.
    H2D copy, forward (CUDA graph) and D2H of neighbouring views overlap (PipelinedCascade).
    init_depth_min / depth_interval: floats shared by the stream (DTU: 425.0 / 2.65)."""
    from .graph import PipelinedCascade
    pipe = None
    keys = []
    n = 0
    for key, imgs, pm in views:
        imgs_h = imgs.unsqueeze(0).contiguous().pin_memory()
        pm_h = pm.unsqueeze(0).contiguous().pin_memory()
        if pipe is None:
            with torch.cuda.device(device):
                pipe = PipelinedCascade(model, imgs_h.to(device), pm_h.to(device),
                                        init_depth_min, depth_interval)
        keys.append(key)
        done = pipe.submit(imgs_h, pm_h)
        if done is not None:
            sink(keys.pop(0), done[0][0].numpy().copy(), done[1][0].numpy().copy())
        n += 1
    if pipe is not None:
        for d, c in pipe.drain():
            sink(keys.pop(0), d[0].numpy().copy(), c[0].numpy().copy())
    return n
