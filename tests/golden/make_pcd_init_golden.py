"""Generate pcd_init.npz by running the reference's own point-cloud initialisation on the CPU.

    python tests/golden/make_pcd_init_golden.py        (needs /root/reference, scipy and PIL)

- GaussianModel.create_from_pcd (gs) and FlatGaussianModel.create_from_pcd (gs_flat) on a ~2k-point cloud: uniform points,
  a cluster, exact duplicates and one isolated point.  `.cuda()` returns the tensor itself and device="cuda" allocations go
  to the CPU, as the other generators map them.
- simple-knn is not part of the reference checkout, so `simple_knn._C.distCUDA2` is stubbed by tests/knn_oracle.py (the
  float32 definition of include/gms_b200.h).  The fixture therefore pins the reference's maths AROUND distCUDA2 -- RGB2SH,
  the clamp, log(sqrt()), the column repeat, the rotation and the opacity -- not distCUDA2 itself.
- readNerfSyntheticInfo on a generated two-view NeRF-synthetic dataset (4x4 RGBA PNGs) after np.random.seed(0), as
  safe_state seeds it: the 100k random points it trains from.  `plyfile` is stubbed by a few lines that keep the structured
  array storePly builds and hand it back to fetchPly, so the f4 / u1 casts are the reference's own numpy.  The first 4096
  rows of points, colours and normals are stored, with a SHA-256 of each full array.
"""
import hashlib
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch
from PIL import Image

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.dirname(HERE))
import knn_oracle  # noqa: E402


def _stub(name, **attrs):
    m = types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


_PLY_FILES = {}


class _PlyElement:
    def __init__(self, data):
        self.data = data

    @staticmethod
    def describe(data, name):
        assert name == "vertex"
        return _PlyElement(data)


class _PlyData:
    def __init__(self, elements):
        self.elements = elements

    def write(self, path):
        _PLY_FILES[path] = self.elements[0].data.copy()

    @staticmethod
    def read(path):
        return {"vertex": _PLY_FILES[path]}


def _dist_cuda2(points):
    return torch.from_numpy(knn_oracle.brute(points.detach().cpu().numpy()))


_stub("plyfile", PlyData=_PlyData, PlyElement=_PlyElement)
_stub("simple_knn")
_stub("simple_knn._C", distCUDA2=_dist_cuda2)
_stub("trimesh")
_stub("smplx")
_stub("smplx.lbs", lbs=None, batch_rodrigues=None, vertices2landmarks=None, find_dynamic_lmk_idx_and_bcoords=None)
_stub("smplx.utils", Struct=object, to_tensor=None, to_np=None, rot_mat_to_euler=None)
_stub("diff_gaussian_rasterization", GaussianRasterizationSettings=object, GaussianRasterizer=object)


def _cpu(fn):
    def f(*a, **k):
        if k.get("device", None) in ("cuda", torch.device("cuda")):
            k["device"] = "cpu"
        return fn(*a, **k)
    return f


for _n in ("zeros", "ones", "empty", "tensor", "full"):
    setattr(torch, _n, _cpu(getattr(torch, _n)))
torch.Tensor.cuda = lambda self, *a, **k: self
# readCamerasFromTransforms builds its RGB image from an np.byte array, which current PIL refuses; older PIL read the bytes
# as uint8, so hand them over that way (the images do not enter the point cloud)
_fromarray = Image.fromarray
Image.fromarray = lambda a, *r, **k: _fromarray(a.view(np.uint8) if a.dtype == np.int8 else a, *r, **k)

from scene.gaussian_model import GaussianModel  # noqa: E402
from games.flat_splatting.scene.flat_gaussian_model import FlatGaussianModel  # noqa: E402
from scene.dataset_readers import readNerfSyntheticInfo  # noqa: E402
from utils.graphics_utils import BasicPointCloud  # noqa: E402

ROWS = 4096


def sha256(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def make_cloud():
    """~2k points: 1500 uniform in [-1,1]^3, 400 in a tight cluster, 100 exact duplicates of uniform points, one far away."""
    rng = np.random.default_rng(5)
    uni = rng.uniform(-1, 1, (1500, 3))
    clu = 0.3 + 0.01 * rng.standard_normal((400, 3))
    dup = uni[rng.choice(1500, 100, replace=False)]
    far = np.array([[40.0, -25.0, 7.5]])
    pts = np.concatenate([uni, clu, dup, far])
    colors = rng.uniform(0, 1, pts.shape)
    return pts, colors


def write_dataset(path):
    frames = []
    for i in range(2):
        os.makedirs(os.path.join(path, "train"), exist_ok=True)
        img = np.zeros((4, 4, 4), np.uint8)
        img[..., i] = 200
        img[..., 3] = 255
        Image.fromarray(img, "RGBA").save(os.path.join(path, "train", f"r_{i}.png"))
        c2w = np.eye(4)
        c2w[:3, 3] = [0.0, -4.0 + 8.0 * i, 0.5]
        frames.append({"file_path": f"./train/r_{i}", "transform_matrix": c2w.tolist()})
    with open(os.path.join(path, "transforms_train.json"), "w") as f:
        json.dump({"camera_angle_x": 0.6911112070083618, "frames": frames}, f)
    with open(os.path.join(path, "transforms_test.json"), "w") as f:
        json.dump({"camera_angle_x": 0.6911112070083618, "frames": []}, f)


def main():
    out = {}
    pts, colors = make_cloud()
    out["pcd_points"], out["pcd_colors"] = pts, colors
    out["pcd_dist2"] = knn_oracle.brute(pts.astype(np.float32))
    for kind, cls in (("gs", GaussianModel), ("gs_flat", FlatGaussianModel)):
        m = cls(3)
        m.create_from_pcd(BasicPointCloud(points=pts, colors=colors, normals=np.zeros_like(pts)), 1.0)
        for n in ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity"):
            out[f"{kind}{n}"] = getattr(m, n).detach().numpy().copy()
        out[f"{kind}_active_sh_degree"] = np.array(m.active_sh_degree)
    with tempfile.TemporaryDirectory() as d:
        write_dataset(d)
        np.random.seed(0)
        info = readNerfSyntheticInfo(d, white_background=True, eval=False)
    pcd = info.point_cloud
    assert pcd is not None
    for n in ("points", "colors", "normals"):
        a = np.asarray(getattr(pcd, n))
        out[f"nerf_{n}"] = a[:ROWS].copy()
        out[f"nerf_{n}_sha256"] = np.array(sha256(a))
        out[f"nerf_{n}_meta"] = np.array(f"{a.dtype.str} {a.shape[0]}x{a.shape[1]}")
    np.savez_compressed(os.path.join(HERE, "pcd_init.npz"), **out)
    print({k: (v.shape, v.dtype) for k, v in out.items()})


if __name__ == "__main__":
    main()
