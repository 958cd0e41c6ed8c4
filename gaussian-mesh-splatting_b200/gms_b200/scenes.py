"""Synthetic cameras, meshes and mesh-Gaussian parameters for tests and bench.py.

Camera conventions restate the reference's (no reference code is imported):
  * world->view matrix, `getWorld2View2`      utils/graphics_utils.py:38-49
  * projection matrix, `getProjectionMatrix`  utils/graphics_utils.py:51-71 (z_sign=+1, z -> [0,1])
  * transposed ("row-vector") storage, full_proj = view^T-stored @ proj^T-stored,
    camera centre = inverse(view)[3,:3]       scene/cameras.py:48-57
  * FoVy derived from FoVx via focal length   utils/graphics_utils.py:73-77
Mesh-Gaussian parameter initialisation follows
  games/mesh_splatting/scene/dataset_readers.py:73-77 (alpha ~ U(0,1)^{F,K,3}),
  games/mesh_splatting/scene/gaussian_mesh_model.py:60-70 (_scale = 1, opacity = inverse_sigmoid(0.1)).
Everything is numpy/torch-CPU; callers move tensors to the GPU.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Tuple

import numpy as np
import torch

NERF_FOVX = 0.6911112070083618  # camera_angle_x of the NeRF-synthetic scenes
ZNEAR, ZFAR = 0.01, 100.0       # scene/cameras.py:48-49
SH_C0 = 0.28209479177387814     # utils/sh_utils.py:26


@dataclass
class Camera:
    """The attributes renderer/gaussian_renderer/__init__.py:39-53 reads from a viewpoint camera."""
    image_width: int
    image_height: int
    FoVx: float
    FoVy: float
    world_view_transform: torch.Tensor  # [4,4], transposed W2C
    full_proj_transform: torch.Tensor   # [4,4]
    camera_center: torch.Tensor         # [3]
    uid: object = None                  # view identity (scene/cameras.py:20 `uid`): keys the per-view statistics of NativeFrame

    @property
    def tanfovx(self) -> float:
        return math.tan(self.FoVx * 0.5)

    @property
    def tanfovy(self) -> float:
        return math.tan(self.FoVy * 0.5)

    def to(self, device) -> "Camera":
        return Camera(self.image_width, self.image_height, self.FoVx, self.FoVy,
                      self.world_view_transform.to(device), self.full_proj_transform.to(device),
                      self.camera_center.to(device), self.uid)


def projection_matrix(znear: float, zfar: float, fovx: float, fovy: float) -> torch.Tensor:
    ty, tx = math.tan(fovy / 2), math.tan(fovx / 2)
    top, right = ty * znear, tx * znear
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (2 * right)
    P[1, 1] = 2.0 * znear / (2 * top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def look_at_camera(eye, target, width: int, height: int, fovx: float = NERF_FOVX,
                   up=(0.0, 0.0, 1.0)) -> Camera:
    """Camera at `eye` looking at `target`; view space is x right, y down, z forward (COLMAP/3DGS)."""
    eye = np.asarray(eye, np.float64)
    target = np.asarray(target, np.float64)
    f = target - eye
    f /= np.linalg.norm(f)
    upv = np.asarray(up, np.float64)
    r = np.cross(f, upv)
    if np.linalg.norm(r) < 1e-8:
        r = np.cross(f, np.array([0.0, 1.0, 0.0]))
    r /= np.linalg.norm(r)
    d = np.cross(f, r)
    Rw2c = np.stack([r, d, f], axis=0)
    Rt = np.eye(4)
    Rt[:3, :3] = Rw2c
    Rt[:3, 3] = -Rw2c @ eye
    w2c = torch.tensor(np.float32(Rt))
    focal = width / (2 * math.tan(fovx / 2))
    fovy = 2 * math.atan(height / (2 * focal))
    wvt = w2c.transpose(0, 1).contiguous()
    proj = projection_matrix(ZNEAR, ZFAR, fovx, fovy).transpose(0, 1)
    full = (wvt.unsqueeze(0).bmm(proj.unsqueeze(0))).squeeze(0).contiguous()
    center = wvt.inverse()[3, :3].contiguous()
    return Camera(width, height, fovx, fovy, wvt, full, center)


def ring_cameras(n: int, radius: float, width: int, height: int, elevation_deg: float = 20.0,
                 fovx: float = NERF_FOVX, phase: float = 0.0) -> List[Camera]:
    cams = []
    el = math.radians(elevation_deg)
    for k in range(n):
        az = phase + 2 * math.pi * k / n
        eye = (radius * math.cos(el) * math.cos(az), radius * math.cos(el) * math.sin(az), radius * math.sin(el))
        cams.append(look_at_camera(eye, (0.0, 0.0, 0.0), width, height, fovx))
    return cams


# --------------------------------------------------------------------------- meshes
def icosphere(level: int, radius: float = 1.0) -> Tuple[np.ndarray, np.ndarray]:
    """Unit icosphere: V = 10*4^level + 2, F = 20*4^level."""
    t = (1.0 + 5 ** 0.5) / 2.0
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2),
         (10, 7, 6), (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11),
         (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    verts = [np.asarray(p, np.float64) / np.linalg.norm(p) for p in v]
    faces = [tuple(x) for x in f]
    for _ in range(level):
        cache = {}
        new_faces = []

        def mid(a, b):
            key = (a, b) if a < b else (b, a)
            if key not in cache:
                m = verts[a] + verts[b]
                verts.append(m / np.linalg.norm(m))
                cache[key] = len(verts) - 1
            return cache[key]

        for a, b, c in faces:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            new_faces += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        faces = new_faces
    return (np.asarray(verts, np.float32) * radius), np.asarray(faces, np.int64)


def grid_surface(nu: int, nv: int, fn, wrap_u=True, wrap_v=True) -> Tuple[np.ndarray, np.ndarray]:
    """Triangulated parametric surface fn(u,v)->xyz on a nu x nv grid; F = 2*nu*nv when both wrap."""
    u = np.arange(nu) / nu if wrap_u else np.linspace(0, 1, nu)
    v = np.arange(nv) / nv if wrap_v else np.linspace(0, 1, nv)
    uu, vv = np.meshgrid(u, v, indexing="ij")
    verts = fn(uu.reshape(-1), vv.reshape(-1)).astype(np.float32)
    iu = np.arange(nu if wrap_u else nu - 1)
    iv = np.arange(nv if wrap_v else nv - 1)
    a, b = np.meshgrid(iu, iv, indexing="ij")
    a = a.reshape(-1); b = b.reshape(-1)
    a1 = (a + 1) % nu; b1 = (b + 1) % nv
    i00 = a * nv + b; i10 = a1 * nv + b; i01 = a * nv + b1; i11 = a1 * nv + b1
    faces = np.concatenate([np.stack([i00, i10, i11], 1), np.stack([i00, i11, i01], 1)], 0)
    return verts, faces.astype(np.int64)


def torus(nu: int, nv: int, R: float = 0.9, r: float = 0.35, center=(0, 0, 0)) -> Tuple[np.ndarray, np.ndarray]:
    c = np.asarray(center, np.float64)

    def fn(u, v):
        a, b = 2 * np.pi * u, 2 * np.pi * v
        return np.stack([(R + r * np.cos(b)) * np.cos(a), (R + r * np.cos(b)) * np.sin(a),
                         r * np.sin(b)], 1) + c

    return grid_surface(nu, nv, fn)


def bumpy_sphere(nu: int, nv: int, radius: float = 0.55, bump: float = 0.08, center=(0, 0, 0)):
    c = np.asarray(center, np.float64)

    def fn(u, v):
        th = 2 * np.pi * u
        ph = np.pi * (0.02 + 0.96 * v)
        rr = radius * (1 + bump * np.sin(5 * th) * np.sin(4 * ph))
        return np.stack([rr * np.sin(ph) * np.cos(th), rr * np.sin(ph) * np.sin(th), rr * np.cos(ph)], 1) + c

    return grid_surface(nu, nv, fn, wrap_u=True, wrap_v=False)


def object_mesh(F_target: int) -> Tuple[np.ndarray, np.ndarray]:
    """Closed 'NeRF-style object': a torus around a bumpy sphere, ~F_target faces in total."""
    half = F_target // 2
    nv = max(8, int(round(math.sqrt(half / 2 / 2.5))))
    nu = max(8, int(round(half / 2 / nv)))
    v1, f1 = torus(nu, nv)
    rem = F_target - f1.shape[0]
    nv2 = max(8, int(round(math.sqrt(rem / 2 / 2))))
    nu2 = max(8, int(round(rem / 2 / (nv2 - 1))))
    v2, f2 = bumpy_sphere(nu2, nv2)
    verts = np.concatenate([v1, v2], 0)
    faces = np.concatenate([f1, f2 + v1.shape[0]], 0)
    return verts.astype(np.float32), faces


# --------------------------------------------------------------------------- parameters
@dataclass
class MeshGaussianParams:
    """Raw (pre-activation) learnable tensors of a gs_mesh model
    (games/mesh_splatting/scene/gaussian_mesh_model.py:59-83, 174-181)."""
    vertices: torch.Tensor        # [V,3]
    faces: torch.Tensor           # [F,3] int64
    _alpha: torch.Tensor          # [F,K,3]
    _scale: torch.Tensor          # [P,1]
    _features_dc: torch.Tensor    # [P,1,3]
    _features_rest: torch.Tensor  # [P,15,3]
    _opacity: torch.Tensor        # [P,1]

    @property
    def P(self) -> int:
        return self._scale.shape[0]

    def to(self, device) -> "MeshGaussianParams":
        return MeshGaussianParams(*[getattr(self, k).to(device) for k in
                                    ("vertices", "faces", "_alpha", "_scale", "_features_dc",
                                     "_features_rest", "_opacity")])

    def learnable(self):
        return [self.vertices, self._alpha, self._scale, self._features_dc, self._features_rest, self._opacity]


def init_mesh_gaussians(verts: np.ndarray, faces: np.ndarray, K: int, seed: int = 0,
                        trained_like: bool = True, sh_coeffs: int = 16) -> MeshGaussianParams:
    g = torch.Generator().manual_seed(seed)
    F = faces.shape[0]
    P = F * K
    alpha = torch.rand(F, K, 3, generator=g)
    scale = torch.ones(P, 1)
    rgb = torch.rand(P, 3, generator=g)
    fdc = ((rgb - 0.5) / SH_C0).reshape(P, 1, 3).contiguous()
    if trained_like:
        frest = 0.05 * torch.randn(P, sh_coeffs - 1, 3, generator=g)
        opacity = 1.0 + 1.5 * torch.randn(P, 1, generator=g)
    else:
        frest = torch.zeros(P, sh_coeffs - 1, 3)
        opacity = torch.full((P, 1), math.log(0.1 / 0.9))
    return MeshGaussianParams(torch.tensor(verts, dtype=torch.float32), torch.tensor(faces, dtype=torch.int64),
                              alpha, scale, fdc, frest, opacity)


def flat_gaussians(P: int, seed: int = 0):
    """BASELINE config 1 inputs: free flat Gaussians (gs_flat), xyz ~ U(-1.3,1.3)^3
    (scene/dataset_readers.py:240; games/flat_splatting/scene/flat_gaussian_model.py:32-35)."""
    g = torch.Generator().manual_seed(seed)
    xyz = (torch.rand(P, 3, generator=g) * 2 - 1) * 1.3
    s12 = torch.exp(math.log(0.02) + 0.3 * torch.randn(P, 2, generator=g))
    scales = torch.cat([torch.full((P, 1), 1e-8), s12], 1)
    q = torch.randn(P, 4, generator=g)
    q = q / q.norm(dim=1, keepdim=True)
    opac = torch.sigmoid(torch.randn(P, 1, generator=g))
    dc = ((torch.rand(P, 1, 3, generator=g) - 0.5) / SH_C0)
    rest = 0.05 * torch.randn(P, 15, 3, generator=g)
    shs = torch.cat([dc, rest], 1).contiguous()
    return dict(means3D=xyz, scales=scales, rotations=q, opacities=opac, shs=shs)


def transform_hotdog_fly(vertices: torch.Tensor, t) -> torch.Tensor:
    """Vertex animation of scripts/render_time_animated.py:34-40 (z += t*sqrt(2 y^2)*0.01)."""
    out = vertices.clone()
    out[:, 2] += t * (vertices[:, 1] ** 2 + vertices[:, 1] ** 2) ** 0.5 * 0.01
    return out


def transform_hotdog(triangles: torch.Tensor, t) -> torch.Tensor:
    """Pseudo-mesh animation of scripts/render_points_time_animated.py:27-30: every triangle vertex moves by
    z += 0.3 sin(pi x + t).  The reference script sweeps t = linspace(0, 10 pi, len(views)) but renders every view at
    t[43] (:44); here `t` is the caller's."""
    out = triangles.clone()
    out[:, :, 2] += 0.3 * torch.sin(triangles[:, :, 0] * math.pi + t)
    return out


def random_point_cloud(num_pts: int = 100_000, seed: int = 0) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The cloud a NeRF-synthetic scene without points3d.ply trains from (readNerfSyntheticInfo, scene/dataset_readers.py:
    233-246, after safe_state's np.random.seed(0); RandomState(seed) draws the same stream): xyz = U * 2.6 - 1.3,
    shs = U / 255, colours SH2RGB(shs).  The reference stores that cloud (storePly) and trains from the file it reads back
    (fetchPly), so it is returned after the same round trip: points cast to float32, and colours truncated to bytes, which
    makes every colour 127/255 (SH2RGB(shs) * 255 lies in [127.5, 127.79)).  -> (points, colors, normals) as fetchPly."""
    from . import io_ply
    rng = np.random.RandomState(seed)
    xyz = rng.random_sample((num_pts, 3)) * 2.6 - 1.3
    shs = rng.random_sample((num_pts, 3)) / 255.0
    return io_ply.point_cloud_arrays(io_ply.point_cloud_elements(xyz, (shs * SH_C0 + 0.5) * 255))


def camera_extent(cams) -> float:
    """scene.cameras_extent: getNerfppNorm's radius (scene/dataset_readers.py:45-66) -- 1.1 times the largest distance of a
    camera centre from their mean.  The arithmetic stays in the centres' dtype, as the reference's numpy keeps it (its
    centres come from getWorld2View2's float32 matrices)."""
    c = np.stack([np.asarray(cam.camera_center.detach().cpu().numpy() if torch.is_tensor(cam.camera_center) else cam.camera_center
                             ).reshape(3, 1) for cam in cams], axis=1)[:, :, 0]
    center = np.mean(c, axis=1, keepdims=True)
    return float(np.max(np.linalg.norm(c - center, axis=0, keepdims=True)) * 1.1)
