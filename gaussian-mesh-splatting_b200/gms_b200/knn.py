"""Mean squared distance to the three nearest other points: simple-knn's distCUDA2 on gms_knn_dist2.

create_from_pcd (scene/gaussian_model.py:124-147, games/flat_splatting/scene/flat_gaussian_model.py:37-60) sets every
Gaussian's initial scale from it.  The result is exact: the fp32 definition in include/gms_b200.h, bit for bit, whatever the
launch order (DESIGN.md 4.4)."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


def mean_dist2(points: torch.Tensor) -> torch.Tensor:
    """points [P,3] (CUDA) -> [P] float32: ((b0 + b1) + b2) / 3 of the three smallest squared distances to other points.
    Scratch comes from the caller's allocator and the call runs on the current stream.  P = 0 gives an empty tensor;
    1 <= P <= 3 and non-finite coordinates raise ValueError (the finiteness check reads one flag back to the host)."""
    if not torch.is_tensor(points):
        raise TypeError("mean_dist2: points must be a tensor")
    if not points.is_cuda:
        raise RuntimeError("mean_dist2: CUDA tensor required (no CPU path in the product)")
    if points.dim() != 2 or points.shape[1] != 3:
        raise ValueError(f"mean_dist2: expected points [P,3]; got {tuple(points.shape)}")
    P = points.shape[0]
    if 1 <= P <= 3:
        raise ValueError(f"mean_dist2: {P} points have no three neighbours each (need P == 0 or P >= 4)")
    if P > 2 ** 31 - 1 - _lib.KNN_BOX:
        raise ValueError("mean_dist2: more than 2^31 - 65 points")
    dev = points.device
    pts = points.detach()
    if pts.dtype != torch.float32 or not pts.is_contiguous():
        pts = pts.float().contiguous()
    out = torch.empty(P, dtype=torch.float32, device=dev)
    if P == 0:
        return out
    if not bool(torch.isfinite(pts).all()):
        raise ValueError("mean_dist2: every coordinate must be finite")
    L = _lib.lib()
    scratch = torch.empty(int(L.gms_knn_scratch_bytes(P)), dtype=torch.uint8, device=dev)
    a = _lib.KnnArgs()
    a.P, a.points, a.dist2, a.scratch, a.scratch_bytes = P, pts.data_ptr(), out.data_ptr(), scratch.data_ptr(), scratch.numel()
    with torch.cuda.device(dev):
        _lib.check(L.gms_knn_dist2(C.byref(a), torch.cuda.current_stream(dev).cuda_stream), "gms_knn_dist2")
    return out
