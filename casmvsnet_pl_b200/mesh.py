"""Mesh a scan on the GPU: TSDF fusion of the filtered depth maps into a sparse voxel volume and
marching-cubes extraction of a coloured triangle mesh (csrc/mesh.cu; float32 / float64 numpy
restatement in oracle/mesh_oracle.py).

    vol = TSDFVolume(points, voxel)          # bricks of 8^3 voxels around the fused points
    vol.integrate(depth, image, P)           # one view or a sequence of views, in order
    verts, colours, faces = vol.extract()    # (N,3) f32, (N,3) u8, (M,3) int32 on the device
    write_mesh_ply("scan.ply", verts, colours, faces)

The truncation distance is TRUNC_VOXELS voxels.  default_voxel_size gives the voxel size the scan
pipeline uses when none is given (eval_pipeline --mesh)."""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from . import _lib

TRUNC_VOXELS = 4
# device bytes per voxel: tsdf, weight, colour (20) + extraction: case (1), triangle count and
# its scan (8), edge flags and their scan (24)
BYTES_PER_VOXEL = 53
MAX_BRICKS = (2 ** 31 - 1) // (512 * 3)
_KEY_NONE = torch.iinfo(torch.int64).max
_CHUNK = 1 << 22          # points per key launch: 8 keys of 8 bytes each, 256 MiB


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check_cuda(name, t, dtype, last_dims):
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype == dtype
            and tuple(t.shape[t.dim() - len(last_dims):]) == tuple(last_dims)):
        raise ValueError(f"{name} must be a {dtype} CUDA tensor of shape (..., "
                         f"{', '.join(map(str, last_dims))})")
    return t.contiguous()


class TSDFVolume:
    """A sparse TSDF volume allocated around `points` ((N,3) float32 CUDA tensor, or a sequence
    of them): every brick of 8^3 voxels that holds a voxel centre within the cube of half-size
    trunc = TRUNC_VOXELS * voxel around a point.  NaN points and points beyond the packable range
    (+-2^23 voxels) are dropped and counted in `dropped`.  Raises CasMVSError when the volume and
    its extraction buffers would not fit in free device memory (or in `max_bytes`), naming a voxel
    size that would."""

    def __init__(self, points, voxel, max_bytes=None):
        if torch.is_tensor(points):
            points = [points]
        points = [_check_cuda("points", p, torch.float32, (3,)).reshape(-1, 3) for p in points]
        if not points:
            raise ValueError("TSDFVolume needs at least one point tensor")
        if not (voxel > 0 and math.isfinite(voxel)):
            raise ValueError(f"voxel size must be > 0, got {voxel}")
        self.device = points[0].device
        self.voxel = float(np.float32(voxel))
        self.trunc = float(np.float32(self.voxel * TRUNC_VOXELS))
        lib = _lib.load()
        self._points = points
        with torch.cuda.device(self.device):
            self.keys, self.dropped = self._brick_keys(self.voxel)
            self._check_fits(max_bytes)
            del self._points
            nvox = self.n_voxels
            self.nbr = torch.empty(self.n_bricks, 7, dtype=torch.int32, device=self.device)
            _lib.check(lib.casmvs_mesh_brick_neighbors(_ptr(self.keys), self.n_bricks,
                                                       _ptr(self.nbr), _stream()),
                       "mesh_brick_neighbors")
            f32 = dict(dtype=torch.float32, device=self.device)
            self.tsdf = torch.zeros(nvox, **f32)
            self.weight = torch.zeros(nvox, **f32)
            self.color = torch.zeros(nvox, 3, **f32)

    @property
    def n_bricks(self):
        return int(self.keys.numel())

    @property
    def n_voxels(self):
        return self.n_bricks * 512

    def _brick_keys(self, voxel):
        """-> (sorted unique keys of the bricks around the points at `voxel`, dropped points)."""
        lib = _lib.load()
        trunc = float(np.float32(voxel * TRUNC_VOXELS))
        dropped = torch.zeros(1, dtype=torch.int64, device=self.device)
        keys = torch.zeros(0, dtype=torch.int64, device=self.device)
        for p in self._points:
            for s in range(0, len(p), _CHUNK):
                c = p[s:s + _CHUNK]
                k = torch.empty(len(c), 8, dtype=torch.int64, device=self.device)
                _lib.check(lib.casmvs_mesh_brick_keys(_ptr(c), len(c), voxel, trunc, _ptr(k),
                                                      _ptr(dropped), _stream()), "mesh_brick_keys")
                keys = torch.unique(torch.cat([keys, torch.unique(k)]))      # sorted
        if len(keys) and int(keys[-1]) == _KEY_NONE:
            keys = keys[:-1]
        return keys.contiguous(), int(dropped.item())

    def _check_fits(self, max_bytes):
        budget = min(device_budget(self.device, max_bytes), MAX_BRICKS * 512 * BYTES_PER_VOXEL)
        need = self.n_voxels * BYTES_PER_VOXEL
        if need <= budget:
            return
        if budget < 512 * BYTES_PER_VOXEL:
            raise _lib.CasMVSError(f"no device memory is left for a TSDF volume ({budget} bytes)")

        def fits(v):
            return len(self._brick_keys(v)[0]) * 512 * BYTES_PER_VOXEL <= budget

        def round_up(x):                         # 3 significant digits, upwards
            e = math.floor(math.log10(x)) - 2
            return float(f"{math.ceil(x / 10.0 ** e)}e{e}")
        # the bricks lie on surfaces: their number falls about with the square of the voxel size
        fit = round_up(float(np.float32(self.voxel * math.sqrt(need / max(budget, 1)))))
        for _ in range(64):
            if fits(float(np.float32(fit))):
                break
            fit = round_up(fit * 1.15)
        raise _lib.CasMVSError(
            f"the TSDF volume at voxel size {self.voxel:.6g} needs {self.n_bricks} bricks "
            f"({need / 2**30:.2f} GiB) but {max(budget, 0) / 2**30:.2f} GiB are available; "
            f"a voxel size of about {fit:g} would fit")

    def integrate(self, depth, image, P):
        """Fuse views in order: depth (H,W) masked depth (0 = none), image (H,W,3) colours, both
        float32 CUDA tensors, P (4,4) world -> pixel; or sequences of those for several views
        (batched on the device, same result as one call per view)."""
        if torch.is_tensor(depth) and depth.dim() == 2:
            depth, image, P = [depth], [image], [P]
        if not (len(depth) == len(image) == len(P)):
            raise ValueError("integrate needs as many images and matrices as depth maps")
        if not len(depth):
            return
        H, W = depth[0].shape
        ds = [_check_cuda("depth", d, torch.float32, (H, W)) for d in depth]
        ims = [_check_cuda("image", i, torch.float32, (H, W, 3)) for i in image]
        Ps = np.ascontiguousarray(np.stack([np.asarray(p, dtype=np.float32).reshape(4, 4) for p in P]))
        arr = ctypes.c_void_p * len(ds)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().casmvs_mesh_integrate(
                _ptr(self.keys), self.n_bricks, self.voxel, self.trunc,
                arr(*[d.data_ptr() for d in ds]), arr(*[i.data_ptr() for i in ims]),
                Ps.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), len(ds), H, W,
                _ptr(self.tsdf), _ptr(self.weight), _ptr(self.color), _stream()), "mesh_integrate")

    def extract(self):
        """Marching cubes -> (verts (N,3) float32, colours (N,3) uint8, faces (M,3) int32) on the
        device, in the same order and bits on every run."""
        with torch.cuda.device(self.device):
            return extract_bricks(self.keys, self.nbr, self.voxel, self.tsdf, self.weight, self.color)


def device_budget(device, max_bytes=None):
    """The bytes a new volume may take on `device`: `max_bytes`, or by default the free device
    memory (counting what torch's allocator holds unused) less a margin of 1 GiB or 5 %."""
    if max_bytes is not None:
        return max_bytes
    free, total = torch.cuda.mem_get_info(device)
    free += torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)
    return free - max(1 << 30, total // 20)


def extract_bricks(keys, nbr, voxel, tsdf, weight, color):
    """Marching cubes over a brick volume (keys (nb,) sorted, nbr (nb,7) from
    casmvs_mesh_brick_neighbors, tsdf / weight (nb*512), color (nb*512,3) float32) on the current
    device -> (verts (N,3) float32, colours (N,3) uint8, faces (M,3) int32)."""
    lib = _lib.load()
    dev, nb = keys.device, int(keys.numel())
    nvox = nb * 512
    i32 = dict(dtype=torch.int32, device=dev)
    cases = torch.empty(nvox, dtype=torch.uint8, device=dev)
    tri_count = torch.empty(nvox, **i32)
    edge_used = torch.empty(nvox * 3, **i32)
    _lib.check(lib.casmvs_mesh_count(_ptr(nbr), nb, _ptr(tsdf), _ptr(weight), _ptr(cases),
                                     _ptr(tri_count), _ptr(edge_used), _stream()), "mesh_count")
    edge_scan = torch.cumsum(edge_used, 0, dtype=torch.int32)
    tri_scan = torch.cumsum(tri_count, 0, dtype=torch.int32)
    n_verts = int(edge_scan[-1]) if nvox else 0
    n_faces = int(tri_scan[-1]) if nvox else 0
    verts = torch.empty(n_verts, 3, dtype=torch.float32, device=dev)
    colours = torch.empty(n_verts, 3, dtype=torch.uint8, device=dev)
    faces = torch.empty(n_faces, 3, **i32)
    if n_faces:
        _lib.check(lib.casmvs_mesh_vertices(
            _ptr(keys), _ptr(nbr), nb, voxel, _ptr(tsdf), _ptr(color), _ptr(edge_used),
            _ptr(edge_scan), _ptr(verts), _ptr(colours), _stream()), "mesh_vertices")
        _lib.check(lib.casmvs_mesh_faces(
            _ptr(nbr), nb, _ptr(cases), _ptr(tri_count), _ptr(tri_scan), _ptr(edge_scan),
            _ptr(faces), _stream()), "mesh_faces")
    return verts, colours, faces


def pixel_footprint(depth, P):
    """World distance between the back-projections through inv(P) of the image-centre pixel
    (W//2, H//2) and its right neighbour at the view's median masked depth (lower median of the
    depths > 0); None when the view has no depth."""
    d = depth[depth > 0]
    if d.numel() == 0:
        return None
    z = float(d.median())
    H, W = depth.shape
    Pinv = np.linalg.inv(np.asarray(P, dtype=np.float64).reshape(4, 4))
    u, v = W // 2, H // 2
    a = Pinv @ np.array([u * z, v * z, z, 1.0])
    b = Pinv @ np.array([(u + 1) * z, v * z, z, 1.0])
    return float(np.linalg.norm(a[:3] / a[3] - b[:3] / b[3]))


def default_voxel_size(depths, Ps):
    """2 x the median over views of pixel_footprint: the voxel size of eval_pipeline --mesh
    without --mesh_voxel."""
    fp = [f for f in (pixel_footprint(d, P) for d, P in zip(depths, Ps)) if f is not None]
    if not fp:
        raise ValueError("no view has a masked depth: cannot derive a voxel size")
    return 2.0 * float(np.median(fp))


def mesh_views(points, depths, images, Ps, voxel=None, max_bytes=None):
    """Volume around `points`, views integrated in order, mesh extracted ->
    (verts, colours, faces, stats dict: voxel, bricks, voxels, vertices, triangles, dropped)."""
    if voxel is None:
        voxel = default_voxel_size(depths, Ps)
    vol = TSDFVolume(points, voxel, max_bytes)
    vol.integrate(list(depths), list(images), list(Ps))
    verts, colours, faces = vol.extract()
    stats = dict(voxel=vol.voxel, bricks=vol.n_bricks, voxels=vol.n_voxels, vertices=len(verts),
                 triangles=len(faces), dropped=vol.dropped)
    return verts, colours, faces, stats


def write_mesh_ply(path, verts, colours, faces):
    """Binary little-endian PLY: the point PLY's vertex layout (float x, y, z, uchar red, green,
    blue) and `element face` with `property list uchar int vertex_indices`."""
    def host(t, dt):
        return np.ascontiguousarray(t.detach().cpu().numpy() if torch.is_tensor(t) else t, dt)
    xyz, rgb, f = host(verts, np.float32), host(colours, np.uint8), host(faces, np.int32)
    v = np.empty(len(xyz), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"),
                                  ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    v["x"], v["y"], v["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    v["red"], v["green"], v["blue"] = rgb[:, 0], rgb[:, 1], rgb[:, 2]
    fr = np.empty(len(f), dtype=[("n", "u1"), ("i", "<i4", (3,))])
    fr["n"] = 3
    fr["i"] = f.reshape(-1, 3)
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {len(xyz)}\nproperty float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\n"
              f"element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        v.tofile(fh)
        fr.tofile(fh)
