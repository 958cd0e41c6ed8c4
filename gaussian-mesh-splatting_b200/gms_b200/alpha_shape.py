"""The editing ("dummy") mesh of a pseudo-mesh: scripts/create_dummy_mesh.py's open3d calls on gms_alpha_shape and
gms_estimate_normals (csrc/gms_alpha.cuh, DESIGN.md 4.11).

    alpha_shape(points, alpha)                          open3d.geometry.TriangleMesh.create_from_point_cloud_alpha_shape
    estimate_normals(points, radius=0.1, max_nn=30)     PointCloud.estimate_normals(KDTreeSearchParamHybrid(radius, max_nn))

Both compute in float64 from float32 points on the GPU.  For points in general position alpha_shape gives open3d's
triangle set; include/gms_b200.h states the tie rule for degenerate input.  Deliberate differences from open3d:
- order: vertices are the referenced points in ascending index, faces have ascending vertex indices and are in
  lexicographic order (open3d's order follows Qhull's facet order);
- exact duplicate points collapse to the lowest index, and nothing else is merged;
- normals have a stated sign, n.(x - mean of the cloud) >= 0 (outward on star-shaped objects); open3d leaves the sign to
  its eigen-solver."""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import _lib


def _points(points: torch.Tensor, what: str) -> torch.Tensor:
    if not torch.is_tensor(points):
        raise TypeError(f"{what}: points must be a tensor")
    if not points.is_cuda:
        raise RuntimeError(f"{what}: CUDA tensor required (no CPU path in the product)")
    if points.dim() != 2 or points.shape[1] != 3:
        raise ValueError(f"{what}: expected points [P,3]; got {tuple(points.shape)}")
    if points.shape[0] >= 2 ** 31 - 1:
        raise ValueError(f"{what}: at most 2^31 - 2 points")
    pts = points.detach()
    if pts.dtype != torch.float32 or not pts.is_contiguous():
        pts = pts.float().contiguous()
    if pts.shape[0] and not bool(torch.isfinite(pts).all()):
        raise ValueError(f"{what}: every coordinate must be finite")
    return pts


def alpha_shape(points: torch.Tensor, alpha: float):
    """points [P,3] (CUDA) -> (vertices float32 [V,3], faces int64 [F,3], index int64 [V]).

    faces index rows of vertices, vertices == points[index] and index is ascending.  Two host synchronisations size the
    neighbour lists and the output; the call runs on the current stream."""
    pts = _points(points, "alpha_shape")
    alpha = float(alpha)
    if not (alpha > 0.0 and math.isfinite(alpha)):
        raise ValueError(f"alpha_shape: alpha must be finite and > 0; got {alpha}")
    dev = pts.device
    bufs = {}

    def _alloc(user, which, nbytes):
        try:
            t = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)
        except Exception:
            return 0
        bufs[int(which)] = t
        return t.data_ptr()

    cb = _lib.ALLOC_FN(_alloc)
    nf, nv = C.c_int64(0), C.c_int64(0)
    a = _lib.AlphaShapeArgs()
    a.P, a.points, a.alpha, a.n_faces, a.n_vertices = pts.shape[0], pts.data_ptr(), alpha, C.pointer(nf), C.pointer(nv)
    L = _lib.lib()
    with torch.cuda.device(dev):
        _lib.check(L.gms_alpha_shape(C.byref(a), cb, None, torch.cuda.current_stream(dev).cuda_stream), "gms_alpha_shape")
    F, V = int(nf.value), int(nv.value)
    if F == 0:
        return (torch.empty(0, 3, dtype=torch.float32, device=dev), torch.empty(0, 3, dtype=torch.int64, device=dev),
                torch.empty(0, dtype=torch.int64, device=dev))
    faces = bufs[_lib.ALPHA_BUF_FACES][:F * 24].view(torch.int64).view(F, 3)
    index = bufs[_lib.ALPHA_BUF_INDEX][:V * 8].view(torch.int64)
    return pts[index], faces, index


def estimate_normals(points: torch.Tensor, radius: float = 0.1, max_nn: int = 30) -> torch.Tensor:
    """points [P,3] (CUDA) -> float32 [P,3] unit normals: the smallest-eigenvalue eigenvector of the covariance of the
    min(max_nn, k) nearest points within radius (the point included), oriented away from the cloud's mean; (0,0,1) where
    k < 3.  Current stream, no host synchronisation after the finiteness check."""
    pts = _points(points, "estimate_normals")
    radius, max_nn = float(radius), int(max_nn)
    if not (radius > 0.0 and math.isfinite(radius)):
        raise ValueError(f"estimate_normals: radius must be finite and > 0; got {radius}")
    if not 1 <= max_nn <= _lib.NORMALS_MAX_NN:
        raise ValueError(f"estimate_normals: max_nn must be in 1..{_lib.NORMALS_MAX_NN}; got {max_nn}")
    dev = pts.device
    P = pts.shape[0]
    out = torch.empty(P, 3, dtype=torch.float32, device=dev)
    if P == 0:
        return out
    L = _lib.lib()
    scratch = torch.empty(int(L.gms_normals_scratch_bytes(P)), dtype=torch.uint8, device=dev)
    a = _lib.NormalsArgs()
    a.P, a.points, a.radius, a.max_nn, a.normals = P, pts.data_ptr(), radius, max_nn, out.data_ptr()
    a.scratch, a.scratch_bytes = scratch.data_ptr(), scratch.numel()
    with torch.cuda.device(dev):
        _lib.check(L.gms_estimate_normals(C.byref(a), torch.cuda.current_stream(dev).cuda_stream), "gms_estimate_normals")
    return out
