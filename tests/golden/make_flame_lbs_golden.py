"""Generate tests/golden/flame_lbs/ by running the REFERENCE's own FLAME class (games/flame_splatting/FLAME/FLAME.py) on a
small synthetic FLAME model file, on the CPU:
  - model_dense.pkl, model_sparse.pkl, model_ch.pkl: one model (V = 10, a 400-column shape basis) written three ways, as
    FLAME's releases are: plain arrays; J_regressor as a pickled scipy.sparse csc_matrix; v_template, shapedirs and
    posedirs as chumpy-style `Ch` objects (a stand-in class under chumpy's module path whose pickled state holds `x`);
  - buffers.npz: FLAME.__init__'s buffers (v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights,
    faces_tensor) for each file, built with smplx.utils' Struct / to_tensor / to_np restated below (smplx is not installed);
  - point_cloud.ply + flame_params.pt: a checkpoint written by GaussianFlameModel.save_ply whose FLAMEPointCloud holds that
    FLAME module, so the pickle carries its buffers under the reference's class paths;
  - expected.npz: FLAME.forward's vertices at random parameters, with smplx.lbs.lbs standing in as tests/flame_lbs_oracle
    (restated from smplx), so the check is of FLAME.forward's own argument handling (the zero padding, the full pose order,
    transl).

    python tests/golden/make_flame_lbs_golden.py
"""
import os
import pickle
import sys
import types

import numpy as np
import scipy.sparse
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import make_ply_golden  # noqa: E402,F401  (module stubs + the reference on sys.path)

import flame_driver  # noqa: E402
import flame_lbs_oracle  # noqa: E402

OUT = os.path.join(HERE, "flame_lbs")


# smplx.utils (public, github.com/vchoutas/smplx): what FLAME.__init__ calls
class Struct:
    def __init__(self, **kwargs):
        for k, v in kwargs.items():
            setattr(self, k, v)


def to_tensor(array, dtype=torch.float32):
    if "torch.tensor" not in str(type(array)):
        return torch.tensor(array, dtype=dtype)


def to_np(array, dtype=np.float32):
    if "scipy.sparse" in str(type(array)):
        array = array.todense()
    return np.array(array, dtype=dtype)


def lbs(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, pose2rot=True):
    """smplx.lbs.lbs for a batch of one, through the restatement."""
    buf = dict(v_template=v_template[0], shapedirs=shapedirs, posedirs=posedirs, J_regressor=J_regressor,
               lbs_weights=lbs_weights, parents=[int(p) for p in parents])
    fp = pose.view(5, 3)
    v = flame_lbs_oracle.lbs(buf, betas[0], torch.zeros(0, dtype=betas.dtype), torch.cat([fp[0], fp[2]]), fp[1],
                             torch.zeros(3, dtype=betas.dtype))
    return v[None], None


chumpy = types.ModuleType("chumpy")
chumpy_ch = types.ModuleType("chumpy.ch")
sys.modules["chumpy"], sys.modules["chumpy.ch"] = chumpy, chumpy_ch


class Ch:
    """Pickles as chumpy's Ch does: the object's __dict__, the array under `x`."""

    def __init__(self, x):
        self.x = x
        self._dirty_vars = set()

    def __array__(self, dtype=None, copy=None):
        return np.asarray(self.x, dtype=dtype)

    @property
    def shape(self):
        return self.x.shape


Ch.__module__ = "chumpy.ch"
chumpy_ch.Ch = Ch

import games.flame_splatting.FLAME  # noqa: E402,F401
from games.flame_splatting.scene.dataset_readers import transform_vertices_function  # noqa: E402
from games.flame_splatting.scene.gaussian_flame_model import GaussianFlameModel  # noqa: E402
from games.flame_splatting.utils.graphics_utils import FLAMEPointCloud  # noqa: E402

FLAME_MODULE = sys.modules["games.flame_splatting.FLAME.FLAME"]
FLAME_MODULE.Struct, FLAME_MODULE.to_tensor, FLAME_MODULE.to_np, FLAME_MODULE.lbs = Struct, to_tensor, to_np, lbs
FLAME_MODULE.vertices2landmarks = lambda *a: torch.zeros(1, 3, 3)      # landmarks: not part of the check


class Config:
    def __init__(self, path, n_shape, n_exp):
        self.flame_model_path = path
        self.static_landmark_embedding_path = os.path.join(OUT, "_static_embedding.pkl")
        self.shape_params, self.expression_params = n_shape, n_exp
        self.use_face_contour = False
        self.use_3D_translation = True
        self.batch_size = 1


def model_dict(rs):
    v, f = flame_driver.uv_sphere(2, 4)
    V = v.shape[0]
    jr = rs.rand(5, V) ** 4
    jr[jr < 0.3] = 0.0
    jr /= jr.sum(1, keepdims=True)
    w = rs.rand(V, 5)
    return dict(v_template=v * 0.1 + 0.003 * rs.randn(V, 3), f=f.astype(np.uint32), shapedirs=rs.randn(V, 3, 400) * 1e-3,
                posedirs=rs.randn(V, 3, 36) * 1e-3, J_regressor=jr, kintree_table=np.array([[2 ** 32 - 1, 0, 1, 1, 1], [0, 1, 2, 3, 4]], np.int64),
                weights=w / w.sum(1, keepdims=True), bs_style="lbs", bs_type="lrotmin")


def main():
    os.makedirs(OUT, exist_ok=True)
    rs = np.random.RandomState(7)
    with open(os.path.join(OUT, "_static_embedding.pkl"), "wb") as fh:
        pickle.dump(dict(lmk_face_idx=np.zeros(3, np.int64), lmk_b_coords=np.full((3, 3), 1 / 3)), fh, protocol=2)
    base = model_dict(rs)
    variants = dict(dense=dict(base),
                    sparse=dict(base, J_regressor=scipy.sparse.csc_matrix(base["J_regressor"]), shapedirs=base["shapedirs"].astype(np.float32)),
                    ch=dict(base, v_template=Ch(base["v_template"]), shapedirs=Ch(base["shapedirs"].astype(np.float32)),
                            posedirs=Ch(base["posedirs"])))
    buffers, flames = {}, {}
    for name, d in variants.items():
        path = os.path.join(OUT, f"model_{name}.pkl")
        with open(path, "wb") as fh:
            pickle.dump(d, fh, protocol=2)
        flame = FLAME_MODULE.FLAME(Config(path, 100, 50))
        flames[name] = flame
        for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "parents", "lbs_weights", "faces_tensor"):
            buffers[f"{name}/{k}"] = getattr(flame, k).numpy()
    os.remove(os.path.join(OUT, "_static_embedding.pkl"))
    flame = flames["dense"]
    torch.manual_seed(3)
    p = dict(shape_params=0.5 * torch.randn(1, 100), expression_params=0.5 * torch.randn(1, 50), pose_params=0.4 * torch.randn(1, 6),
             neck_pose=0.4 * torch.randn(1, 3), transl=0.05 * torch.randn(1, 3))
    with torch.no_grad():
        verts, _ = flame(**p)
    expected = {k: v.numpy() for k, v in p.items()}
    expected["vertices"] = verts[0].numpy()

    # a checkpoint written by the reference's save_ply, its FLAMEPointCloud holding the FLAME module
    V, F, K = flame.v_template.shape[0], flame.faces_tensor.shape[0], 2
    m = GaussianFlameModel(0)
    z = lambda n: torch.zeros(1, n)
    m.point_cloud = FLAMEPointCloud(alpha=None, points=None, colors=None, normals=None, faces=flame.faces_tensor, vertices_init=None,
                                    flame_model=flame, transform_vertices_function=transform_vertices_function,
                                    flame_model_shape_init=z(100), flame_model_expression_init=z(50), flame_model_pose_init=z(6),
                                    flame_model_neck_pose_init=z(3), flame_model_transl_init=z(3), vertices_enlargement_init=8.35)
    m._flame_shape, m._flame_exp, m._flame_pose = (torch.nn.Parameter(p[k].clone()) for k in ("shape_params", "expression_params", "pose_params"))
    m._flame_neck_pose, m._flame_trans = torch.nn.Parameter(p["neck_pose"].clone()), torch.nn.Parameter(p["transl"].clone())
    m._vertices_enlargement = torch.nn.Parameter(8.35 * torch.ones(V, 3))
    m.faces = flame.faces_tensor
    m._alpha = torch.nn.Parameter(torch.randn(F, K, 3))
    m._scales = torch.nn.Parameter(0.5 + torch.rand(F * K, 1))
    m._opacity = torch.nn.Parameter(torch.randn(F * K, 1))
    m._features_dc = torch.nn.Parameter(torch.randn(F * K, 1, 3))
    m._features_rest = torch.nn.Parameter(torch.zeros(F * K, 0, 3))
    m.save_ply(os.path.join(OUT, "point_cloud.ply"))
    np.savez_compressed(os.path.join(OUT, "buffers.npz"), **buffers)
    np.savez_compressed(os.path.join(OUT, "expected.npz"), **expected)
    for name in sorted(os.listdir(OUT)):
        print(name, os.path.getsize(os.path.join(OUT, name)))


if __name__ == "__main__":
    main()
