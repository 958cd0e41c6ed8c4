"""Generate tests/golden/flame/{point_cloud.ply, flame_params.pt, expected.npz} by running the REFERENCE's own
GaussianFlameModel (games/flame_splatting/scene/gaussian_flame_model.py) on the CPU:
  - update_alpha + prepare_scaling_rot with a stub FLAME model that returns fixed leaf vertices [1,V,3], transformed by the
    reference's own transform_vertices_function (games/flame_splatting/scene/dataset_readers.py:40-45);
  - autograd gradients of _alpha, _scales, the stub's raw vertices and _vertices_enlargement for a fixed upstream gradient
    on (_xyz, _scaling, _rotation);
  - a checkpoint written by its save_ply (:230-252), whose FLAMEPointCloud holds the stub under FLAME's class path
    (games.flame_splatting.FLAME.FLAME.FLAME), so the pickle names the classes the reference's checkpoints name.
The module stubs (plyfile writer, smplx, simple_knn, ...) are make_ply_golden.py's.

    python tests/golden/make_flame_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import make_ply_golden  # noqa: E402,F401  (module stubs + the reference on sys.path)
import games.flame_splatting.FLAME  # noqa: E402,F401
from games.flame_splatting.scene.dataset_readers import transform_vertices_function  # noqa: E402
from games.flame_splatting.scene.gaussian_flame_model import GaussianFlameModel  # noqa: E402
from games.flame_splatting.utils.graphics_utils import FLAMEPointCloud  # noqa: E402

import flame_driver  # noqa: E402

OUT = os.path.join(HERE, "flame")
FLAME_MODULE = sys.modules["games.flame_splatting.FLAME.FLAME"]


class FLAME:
    """Stub with FLAME.forward's signature: returns its fixed leaf vertices [1,V,3]."""

    def __init__(self, v):
        self.v = v

    def __call__(self, shape_params=None, expression_params=None, pose_params=None, neck_pose=None, transl=None):
        return self.v, None


FLAME.__module__ = FLAME_MODULE.__name__


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(11)
    rs = np.random.RandomState(3)
    v, f = flame_driver.uv_sphere(5, 6)
    v = (v * 0.1 + 0.004 * rs.randn(*v.shape)).astype(np.float32)
    V, F, K = v.shape[0], f.shape[0], 4
    P = F * K
    raw = torch.nn.Parameter(torch.tensor(v)[None])
    stub = FLAME(raw)
    real = FLAME_MODULE.FLAME
    FLAME_MODULE.FLAME = FLAME          # pickled under FLAME's class path
    try:
        m = GaussianFlameModel(3)
        z = lambda n: torch.zeros(1, n)
        enl = torch.tensor((8.35 * (1 + 0.05 * rs.randn(V, 3))).astype(np.float32))
        m.point_cloud = FLAMEPointCloud(alpha=None, points=None, colors=None, normals=None, faces=torch.tensor(f), vertices_init=None,
                                        flame_model=stub, transform_vertices_function=transform_vertices_function,
                                        flame_model_shape_init=z(100), flame_model_expression_init=z(50), flame_model_pose_init=z(6),
                                        flame_model_neck_pose_init=z(3), flame_model_transl_init=z(3), vertices_enlargement_init=8.35)
        m._flame_shape, m._flame_exp, m._flame_pose = (torch.nn.Parameter(0.1 * torch.randn(1, n)) for n in (100, 50, 6))
        m._flame_neck_pose, m._flame_trans = torch.nn.Parameter(0.1 * torch.randn(1, 3)), torch.nn.Parameter(0.1 * torch.randn(1, 3))
        m._vertices_enlargement = torch.nn.Parameter(enl)
        m.faces = torch.tensor(f)
        a = 2.0 * torch.randn(F, K, 3)
        a[0, 0] = torch.tensor([1e3, 0.0, -1e3])
        a[0, 1] = 0.5
        m._alpha = torch.nn.Parameter(a)
        m._scales = torch.nn.Parameter(0.5 + torch.rand(P, 1))
        m._opacity = torch.nn.Parameter(torch.randn(P, 1))
        m._features_dc = torch.nn.Parameter(torch.randn(P, 1, 3))
        m._features_rest = torch.nn.Parameter(0.1 * torch.randn(P, 15, 3))
        m.update_alpha()
        m.prepare_scaling_rot()
        u = [torch.tensor(rs.randn(*t.shape).astype(np.float32)) for t in (m._xyz, m._scaling, m._rotation)]
        ((m._xyz * u[0]).sum() + (m._scaling * u[1]).sum() + (m._rotation * u[2]).sum()).backward()
        d = lambda t: t.detach().numpy()
        expected = dict(raw_vertices=d(raw)[0], faces=f, _alpha=d(m._alpha), _scales=d(m._scales), _opacity=d(m._opacity),
                        _features_dc=d(m._features_dc), _features_rest=d(m._features_rest), _vertices_enlargement=d(enl),
                        vertices=d(m.vertices), alpha=d(m.alpha), _xyz=d(m._xyz), _scaling=d(m._scaling), _rotation=d(m._rotation),
                        up_xyz=d(u[0]), up_scaling=d(u[1]), up_rotation=d(u[2]), d_alpha=d(m._alpha.grad), d_scales=d(m._scales.grad),
                        d_raw_vertices=d(raw.grad)[0], d_vertices_enlargement=d(m._vertices_enlargement.grad))
        for n in ("_flame_shape", "_flame_exp", "_flame_pose", "_flame_neck_pose", "_flame_trans"):
            expected[n] = d(getattr(m, n))
        m.save_ply(os.path.join(OUT, "point_cloud.ply"))   # the reference's writer: update_alpha, prepare_scaling_rot, _save_ply, torch.save
    finally:
        FLAME_MODULE.FLAME = real
    np.savez_compressed(os.path.join(OUT, "expected.npz"), **expected)
    for name in sorted(os.listdir(OUT)):
        print(name, os.path.getsize(os.path.join(OUT, name)))


if __name__ == "__main__":
    main()
