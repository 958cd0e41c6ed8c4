"""Generate tests/golden/multi_mesh_ply/{point_cloud.ply, model_params.pt, expected.npz} by running the REFERENCE's own
GaussianMultiMeshModel.save_ply (games/multi_mesh_splatting/scene/gaussian_multi_mesh_model.py:222-243 ->
GaussianModel._save_ply) on a two-mesh model with K = (2, 3) splats per face.  Property order, the per-mesh LISTS of
model_params.pt and the pickled `point_cloud` entries (MultiMeshPointCloud named tuples, as the reference's reader builds them,
games/multi_mesh_splatting/scene/dataset_readers.py:66-102) therefore come from the reference's code; the PLY container is
written by make_ply_golden.py's `plyfile` stand-in.

    python tests/golden/make_multi_mesh_ply_golden.py
"""
import os

import numpy as np
import torch

import make_ply_golden  # noqa: F401  (module stubs, sys.path)
from games.multi_mesh_splatting.scene.gaussian_multi_mesh_model import GaussianMultiMeshModel  # noqa: E402
from games.multi_mesh_splatting.utils.graphics_utils import MultiMeshPointCloud  # noqa: E402
from gms_b200 import scenes  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "multi_mesh_ply")


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(7)
    m = GaussianMultiMeshModel(3)
    vs, fs, als, scs, pcds = [], [], [], [], []
    for k, (lvl, K) in enumerate([(0, 2), (1, 3)]):
        v, f = scenes.icosphere(lvl, radius=0.5 + 0.3 * k)
        v = (v + np.float32([1.5 * k, 0, 0]) + 0.02 * np.random.RandomState(k).randn(*v.shape)).astype(np.float32)
        F = f.shape[0]
        vs.append(torch.nn.Parameter(torch.tensor(v)))
        fs.append(torch.tensor(f).long())
        als.append(torch.nn.Parameter(torch.rand(F, K, 3)))
        scs.append(torch.nn.Parameter(0.5 + torch.rand(F * K, 1)))
        tri = torch.tensor(v)[torch.tensor(f).long()]
        pcds.append(MultiMeshPointCloud(alpha=als[-1].detach().clone(), points=torch.matmul(als[-1].detach(), tri).reshape(-1, 3),
                                        colors=np.zeros((F * K, 3)), normals=np.zeros((F * K, 3)), vertices=v, faces=f, triangles=tri))
    P = sum(s.shape[0] for s in scs)
    m.vertices, m.faces, m._alpha, m._scale, m.point_cloud = vs, fs, als, scs, pcds
    m._opacity = torch.nn.Parameter(torch.randn(P, 1))
    m._features_dc = torch.nn.Parameter(torch.randn(P, 1, 3))
    m._features_rest = torch.nn.Parameter(torch.randn(P, 15, 3))
    ply = os.path.join(OUT, "point_cloud.ply")
    m.save_ply(ply)                       # the reference's writer: update_alpha, prepare_scaling_rot, _save_ply, torch.save
    out = dict(n_mesh=np.int64(2), _opacity=m._opacity.detach().numpy(), _features_dc=m._features_dc.detach().numpy(),
               _features_rest=m._features_rest.detach().numpy(), _xyz=m._xyz.detach().numpy(), _scaling=m._scaling.detach().numpy(),
               _rotation=m._rotation.detach().numpy())
    for k in range(2):
        out[f"vertices{k}"] = vs[k].detach().numpy(); out[f"faces{k}"] = fs[k].numpy()
        out[f"_alpha{k}"] = als[k].detach().numpy(); out[f"_scale{k}"] = scs[k].detach().numpy()
    np.savez_compressed(os.path.join(OUT, "expected.npz"), **out)
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
