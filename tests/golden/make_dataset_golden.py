"""Generate dataset.npz by running the reference's own scene loading on the CPU over the datasets of tests/dataset_cases.py.

    python tests/golden/make_dataset_golden.py        (needs /root/reference and PIL)

For every case of dataset_cases.CASES, in a fresh copy of its dataset (the reference writes points3d.ply / points3D.ply into
the source directory):
- random.seed(0), np.random.seed(0), torch.manual_seed(0) as safe_state does; then readNerfSyntheticInfo,
  readNerfSyntheticMeshInfo (gs_mesh) or readColmapSceneInfo; Scene.__init__'s shuffle of the train and test infos
  (scene/__init__.py:84-86) and cameraList_from_camInfos (loadCam, PILtoTorch) with data_device "cpu"; then 40 iterations
  of train.py's viewpoint_stack.pop(randint(0, len - 1)) on the same `random` stream.  For gs_mesh,
  GaussianMeshModel.create_from_pcd on the scene's cloud gives the initial tensors.
- Stubs: `plyfile` keeps the structured array storePly builds in memory and hands it back to fetchPly (the f4 / u1 casts are
  the reference's own numpy); `trimesh.load` parses the OBJ's `v` / `f` records into float64 vertices and int64 faces
  (the fixture mesh has no duplicate vertices, so trimesh's merging would not change it); `.cuda()` returns the tensor
  itself and device="cuda" allocations go to the CPU; simple-knn, smplx and the rasterizer are empty modules.
  readCamerasFromTransforms builds its RGB image from an np.byte array, which current PIL refuses; older PIL read the bytes
  as uint8, so they are handed over that way.
Stored per case: R, T, FoVs, sizes, world_view_transform, full_proj_transform, camera_center, names (train / test, in
shuffled order), cameras_extent, the view order, every ground-truth image as bytes (PILtoTorch * 255, checked exact), the
point cloud (the first 256 rows and a SHA-256 of each full array) or the gs_mesh tensors.
"""
import hashlib
import os
import random
import shutil
import sys
import tempfile
import types

import numpy as np
import torch
from PIL import Image

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "gaussian-mesh-splatting_b200"))
import dataset_cases  # noqa: E402


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
        if path not in _PLY_FILES:      # a points3d.ply that came with the dataset
            from gms_b200 import io_ply
            _PLY_FILES[path] = io_ply.read_ply_vertices(path)[0]
        return {"vertex": _PLY_FILES[path]}


class _Mesh:
    def __init__(self, path):
        v, f = [], []
        for line in open(path):
            p = line.split()
            if p and p[0] == "v":
                v.append([float(x) for x in p[1:4]])
            elif p and p[0] == "f":
                f.append([int(x) - 1 for x in p[1:4]])
        self.vertices, self.faces = np.array(v, np.float64), np.array(f, np.int64)


_stub("plyfile", PlyData=_PlyData, PlyElement=_PlyElement)
_stub("simple_knn")
_stub("simple_knn._C", distCUDA2=None)
_stub("trimesh", load=lambda path, force=None: _Mesh(path))
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
_fromarray = Image.fromarray
Image.fromarray = lambda a, *r, **k: _fromarray(a.view(np.uint8) if a.dtype == np.int8 else a, *r, **k)

from scene.dataset_readers import readColmapSceneInfo, readNerfSyntheticInfo  # noqa: E402
from games.mesh_splatting.scene.dataset_readers import readNerfSyntheticMeshInfo  # noqa: E402
from games.mesh_splatting.scene.gaussian_mesh_model import GaussianMeshModel  # noqa: E402
from utils.camera_utils import cameraList_from_camInfos  # noqa: E402

ROWS, ORDER = 256, 40


def sha256(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def run_case(src: str, kw: dict, out: dict, key: str) -> None:
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    if os.path.exists(os.path.join(src, "sparse")):
        info = readColmapSceneInfo(src, "images", kw["eval"])
    elif kw["gs_type"] == "gs_mesh":
        info = readNerfSyntheticMeshInfo(src, kw["white_background"], kw["eval"], kw["num_splats"])
    else:
        info = readNerfSyntheticInfo(src, kw["white_background"], kw["eval"])
    random.shuffle(info.train_cameras)
    random.shuffle(info.test_cameras)
    args = types.SimpleNamespace(resolution=kw["resolution"], data_device="cpu")
    out[f"{key}/extent"] = np.array(info.nerf_normalization["radius"], np.float64)
    for split, infos in (("train", info.train_cameras), ("test", info.test_cameras)):
        cams = cameraList_from_camInfos(infos, 1.0, args)
        out[f"{key}/{split}/names"] = np.array([c.image_name for c in cams], dtype="U64")
        out[f"{key}/{split}/R"] = np.array([c.R for c in cams], np.float64).reshape(-1, 3, 3)
        out[f"{key}/{split}/T"] = np.array([c.T for c in cams], np.float64).reshape(-1, 3)
        out[f"{key}/{split}/fov"] = np.array([[c.FoVx, c.FoVy] for c in cams], np.float64).reshape(-1, 2)
        out[f"{key}/{split}/size"] = np.array([[c.image_width, c.image_height] for c in cams], np.int64).reshape(-1, 2)
        for n in ("world_view_transform", "full_proj_transform", "camera_center"):
            out[f"{key}/{split}/{n}"] = np.array([getattr(c, n).numpy() for c in cams], np.float32)
        for i, c in enumerate(cams):
            x = c.original_image.numpy()
            b = np.round(x * 255.0).astype(np.uint8)
            assert np.array_equal(torch.from_numpy(b).float().numpy() / 255.0, x.astype(np.float64)) or \
                np.array_equal((torch.from_numpy(b) / 255.0).numpy(), x), "image is not bytes / 255"
            out[f"{key}/{split}/image{i}"] = b.transpose(1, 2, 0).copy()      # [H,W,3]
    stack, order = [], []
    n = len(info.train_cameras)
    for _ in range(ORDER):
        if not stack:
            stack = list(range(n))
        order.append(stack.pop(random.randint(0, len(stack) - 1)))
    out[f"{key}/order"] = np.array(order, np.int64)
    if kw["gs_type"] == "gs_mesh":
        m = GaussianMeshModel(3)
        m.create_from_pcd(info.point_cloud, info.nerf_normalization["radius"])
        for nme in ("vertices", "faces", "_alpha", "_scale", "_features_dc", "_features_rest", "_opacity"):
            out[f"{key}/mesh{nme}"] = getattr(m, nme).detach().numpy().copy()
    else:
        pcd = info.point_cloud
        for nme in ("points", "colors", "normals"):
            a = np.asarray(getattr(pcd, nme))
            out[f"{key}/pcd_{nme}"] = a[:ROWS].copy()
            out[f"{key}/pcd_{nme}_sha256"] = np.array(sha256(a))
            out[f"{key}/pcd_{nme}_meta"] = np.array(f"{a.dtype.str} {a.shape[0]}x{a.shape[1]}")


def main():
    out = {}
    with tempfile.TemporaryDirectory() as d:
        dirs = dataset_cases.write_all(os.path.join(d, "src"))
        for key, (ds, kw) in dataset_cases.CASES.items():
            work = os.path.join(d, "work", key)
            shutil.copytree(dirs[ds], work)
            run_case(work, kw, out, key)
    np.savez_compressed(os.path.join(HERE, "dataset.npz"), **out)
    print(f"{len(out)} arrays, {os.path.getsize(os.path.join(HERE, 'dataset.npz'))} bytes")


if __name__ == "__main__":
    main()
