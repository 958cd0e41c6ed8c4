"""Point clouds for the alpha-shape tests and tools/alpha_shape_eval.py.

surface_flat_gaussians: gs_flat Gaussians laid flat on scenes.object_mesh surfaces (the flat axis along the face normal, the
two in-plane scales log-normal around `scale`), so the pseudo-mesh's neighbourhoods resemble a trained model's."""
from __future__ import annotations

import numpy as np
import torch

from gms_b200 import scenes


def _quat_from_matrix(R: np.ndarray) -> np.ndarray:
    """[N,3,3] rotations -> [N,4] (w, x, y, z), build_rotation's convention."""
    w = np.sqrt(np.maximum(0.0, 1 + R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2])) / 2
    x = np.sqrt(np.maximum(0.0, 1 + R[:, 0, 0] - R[:, 1, 1] - R[:, 2, 2])) / 2
    y = np.sqrt(np.maximum(0.0, 1 - R[:, 0, 0] + R[:, 1, 1] - R[:, 2, 2])) / 2
    z = np.sqrt(np.maximum(0.0, 1 - R[:, 0, 0] - R[:, 1, 1] + R[:, 2, 2])) / 2
    x = np.copysign(x, R[:, 2, 1] - R[:, 1, 2])
    y = np.copysign(y, R[:, 0, 2] - R[:, 2, 0])
    z = np.copysign(z, R[:, 1, 0] - R[:, 0, 1])
    q = np.stack([w, x, y, z], 1)
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def surface_flat_gaussians(n: int, seed: int = 0, scale: float = 0.004, faces: int = 20000):
    """dict(xyz [n,3], scaling [n,2] log-scales, rotation [n,4], features_dc [n,1,3], features_rest [n,15,3], opacity [n,1])."""
    rng = np.random.default_rng(seed)
    V, F = scenes.object_mesh(faces)
    V = V.astype(np.float64)
    tri = V[F]
    area = 0.5 * np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
    f = rng.choice(len(F), size=n, p=area / area.sum())
    r1, r2 = rng.random(n), rng.random(n)
    s = np.sqrt(r1)
    t = tri[f]
    xyz = (1 - s)[:, None] * t[:, 0] + (s * (1 - r2))[:, None] * t[:, 1] + (s * r2)[:, None] * t[:, 2]
    nrm = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    a = rng.standard_normal((n, 3))
    t1 = a - (a * nrm).sum(1, keepdims=True) * nrm
    t1 /= np.linalg.norm(t1, axis=1, keepdims=True)
    t2 = np.cross(nrm, t1)
    q = _quat_from_matrix(np.stack([nrm, t1, t2], 2))          # columns: the flat axis, then the two in-plane axes
    scaling = np.log(scale) + 0.3 * rng.standard_normal((n, 2))
    g = torch.Generator().manual_seed(seed)
    f32 = lambda x: torch.tensor(x, dtype=torch.float32)
    return dict(xyz=f32(xyz), scaling=f32(scaling), rotation=f32(q),
                features_dc=((torch.rand(n, 1, 3, generator=g) - 0.5) / 0.28209479177387814),
                features_rest=0.05 * torch.randn(n, 15, 3, generator=g), opacity=torch.randn(n, 1, generator=g))


def pseudomesh_points(n: int, seed: int = 0, scale: int = 2, device="cuda") -> torch.Tensor:
    """The [3n,3] float32 points create_dummy_mesh.py builds from the pseudo-mesh of surface_flat_gaussians(n): triangles
    (PointsModel.from_gaussians, on the GPU) reshaped and times `scale`."""
    from gms_b200.model import PointsModel
    g = surface_flat_gaussians(n, seed)
    tri = PointsModel.from_gaussians(g["xyz"], g["scaling"], g["rotation"], g["features_dc"], g["features_rest"], g["opacity"],
                                     device).triangles
    return (tri.reshape(3 * n, 3) * scale).contiguous()


def box(n: int, seed: int) -> np.ndarray:
    return np.random.default_rng(seed).random((n, 3)).astype(np.float32)


def shell(n: int, seed: int, noise: float = 0.02) -> np.ndarray:
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, 3))
    return (x / np.linalg.norm(x, axis=1, keepdims=True) * (1 + noise * rng.standard_normal((n, 1)))).astype(np.float32)

