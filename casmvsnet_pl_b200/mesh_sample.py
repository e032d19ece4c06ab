"""Uniform surface sampling of a triangle mesh on the GPU, so that the point-cloud scorers
(dtu_eval, tnt_eval) can score a mesh (csrc/mesh_sample.cu; numpy float64 restatement in
oracle/mesh_sample_oracle.py, bit for bit).

    samples = sample_surface(verts, faces, spacing)      # (S,3) float32 on the device

The rule (include/casmvs.h states every operation): face (a, b, c), in its stored corner order,
with L its longest edge in double, is cut into n = max(1, ceil(L / spacing)) rows (clamped at
2^16) and sampled on the lattice (a + (i/n)(b - a)) + (j/n)(c - a), i = 0..n, j = 0..n - i:
(n + 1)(n + 2) / 2 samples, no two of a face farther than `spacing` from their neighbours.
Samples are face-major, then row-major in (i, j).  Shared edges and vertices are sampled once
per face that holds them and the duplicates are kept; vertices no face uses are not sampled."""
from __future__ import annotations

import ctypes
import math
import os

import numpy as np
import torch

from . import _lib, io, mesh

# device bytes per sample while a mesh is scored: the sample itself (12) and the scorers'
# per-point working set (cell keys, sort order and its scratch, the sorted copy, visiting ranks
# and states).  The largest peak allocation per sample bench_mesh_eval.py measured, 115.7 bytes
# on the 1 % decimated DTU-sized mesh (H100 80GB HBM3), rounded up
BYTES_PER_SAMPLE = 116
MAX_SAMPLES = 2 ** 31            # the pcd_* kernels take int counts


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(verts, faces, spacing):
    if isinstance(spacing, bool) or not isinstance(spacing, (int, float, np.floating, np.integer)) \
            or not (math.isfinite(spacing) and spacing > 0):
        raise ValueError(f"spacing must be a finite number > 0, got {spacing!r}")
    for name, t, dtypes in (("verts", verts, (torch.float32,)),
                            ("faces", faces, (torch.int32, torch.int64))):
        if not (torch.is_tensor(t) and t.dtype in dtypes and t.dim() == 2 and t.shape[1] == 3):
            raise ValueError(f"{name} must be a tensor of shape (N, 3) and dtype "
                             f"{' or '.join(map(str, dtypes))}")
    if len(faces) == 0:
        raise ValueError("the mesh has no faces: there is no surface to sample")
    if 3 * max(len(verts), len(faces)) >= 2 ** 31:
        raise ValueError(f"a mesh of {len(verts)} vertices and {len(faces)} faces is too large "
                         "(3 x either must stay below 2^31)")
    if not bool(torch.isfinite(verts).all()):
        raise ValueError("verts holds a non-finite coordinate")
    if not bool(((faces >= 0) & (faces < len(verts))).all()):
        raise ValueError(f"faces holds an index outside 0..{len(verts) - 1}")
    if not (verts.is_cuda and faces.is_cuda and verts.device == faces.device):
        raise ValueError("surface sampling runs on the GPU: verts and faces must be CUDA tensors "
                         "on one device")


def sample_counts(verts, faces, spacing):
    """-> (n (F,) int32, count (F,) int64, start (F,) int64 exclusive prefix sum) on the device.
    Inputs are checked by the caller."""
    F = len(faces)
    n = torch.empty(F, dtype=torch.int32, device=verts.device)
    count = torch.empty(F, dtype=torch.int64, device=verts.device)
    _lib.check(_lib.load().casmvs_mesh_sample_count(_ptr(verts), _ptr(faces), F, float(spacing),
                                                    _ptr(n), _ptr(count), _stream()),
               "mesh_sample_count")
    start = torch.cumsum(count, 0) - count
    return n, count, start


def sample_points(verts, faces, n, start, S):
    """The points kernel alone -> (S,3) float32."""
    out = torch.empty(S, 3, dtype=torch.float32, device=verts.device)
    _lib.check(_lib.load().casmvs_mesh_sample_points(_ptr(verts), _ptr(faces), len(faces), _ptr(n),
                                                     _ptr(start), S, _ptr(out), _stream()),
               "mesh_sample_points")
    return out


def sample_surface(verts, faces, spacing, max_bytes=None):
    """Samples of the surface of (verts (V,3) float32, faces (F,3) int32 or int64) CUDA tensors at
    `spacing` -> (S,3) float32 CUDA tensor (the rule is the module's).  Refuses a spacing that is
    not finite and > 0, an empty face list, non-finite vertices, out-of-range indices, S >= 2^31
    and, with CasMVSError, work over mesh.device_budget (BYTES_PER_SAMPLE per sample), all before
    a sample buffer is allocated."""
    _check(verts, faces, spacing)
    dev = verts.device
    with torch.cuda.device(dev):
        v = verts.contiguous()
        f = faces.int().contiguous()
        n, count, start = sample_counts(v, f, spacing)
        S = int(count.sum())
        if S >= MAX_SAMPLES:
            raise ValueError(f"{len(f)} faces at spacing {spacing:g} make {S} samples; the scorers "
                             f"take fewer than 2^31 points: use a coarser spacing")
        need = S * BYTES_PER_SAMPLE
        budget = mesh.device_budget(dev, max_bytes)
        if need > budget:
            raise _lib.CasMVSError(
                f"scoring {S} surface samples needs {need} bytes of device memory "
                f"({BYTES_PER_SAMPLE} per sample) but {max(budget, 0)} bytes are available")
        return sample_points(v, f, n, start, S)


def load_mesh(mesh_or_ply, device):
    """(verts, faces) CUDA tensors as given, or a mesh PLY (io.read_mesh_ply) read to `device`.
    A PLY without faces is refused, naming the file."""
    if isinstance(mesh_or_ply, (str, os.PathLike)):
        v, _, f = io.read_mesh_ply(mesh_or_ply)
        if len(f) == 0:
            raise ValueError(f"{mesh_or_ply}: the mesh PLY has no faces")
        dev = torch.device(device)
        if dev.type != "cuda" or not torch.cuda.is_available():
            raise _lib.CasMVSError("mesh scoring runs on the GPU (no CPU fallback)")
        return (torch.from_numpy(np.ascontiguousarray(v)).to(dev),
                torch.from_numpy(np.ascontiguousarray(f)).to(dev))
    if isinstance(mesh_or_ply, (tuple, list)) and len(mesh_or_ply) == 2:
        return mesh_or_ply
    raise TypeError("mesh must be (verts, faces) CUDA tensors or a mesh PLY path")
