"""Generate train_mesh_types.npz: what the reference's gs_multi_mesh and gs_flame scene readers and train.py's output
directory set-up produce, from the reference's own code, on the CPU.

    python tests/golden/make_train_mesh_types_golden.py        (needs /root/reference and PIL)

Importing make_cli_golden installs make_dataset_golden's stubs (plyfile in memory, CUDA allocations and `.cuda()` on the
CPU, empty simple-knn / smplx / rasterizer modules); importing make_flame_lbs_golden gives the reference's FLAME class
smplx.utils' helpers and smplx.lbs.lbs (restated, tests/flame_lbs_oracle.py) with the landmarks stubbed, and
make_ply_golden's plyfile writer the file bytes of a stored cloud.  `trimesh.load` is a stand-in that returns the OBJ's
`v` / `f` records as written, with triangles = vertices[faces].  Then, on the scenes of tests/mesh_types_cases.py:
- random.seed(0), np.random.seed(0), torch.manual_seed(0) as safe_state does, then readColmapMeshSceneInfo(--meshes a b
  --num_splats 2 3, --eval) or readNerfSyntheticFlameInfo (FlameConfig pointed at tests/golden/flame_lbs/model_dense.pkl),
  Scene.__init__'s shuffle of the train and test infos and cameraList_from_camInfos.
- Stored: per split the names, R, T, FoVs and sizes in shuffled order, cameras_extent; per mesh `alpha` and `colors` of the
  reader's point cloud and the bytes of points3d_<i>.ply; for FLAME `alpha`, `colors`, the transformed initial vertices,
  the faces and the rows of points3d.ply.
- cfg_args: make_cli_golden.reference_cfg_args for a gs_multi_mesh and a gs_flame command line."""
import os
import random
import shutil
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_cli_golden as mcg  # noqa: E402  (installs make_dataset_golden's stubs, imports the reference's train.py)
import make_flame_lbs_golden as mflg  # noqa: E402  (FLAME's smplx helpers)
import make_ply_golden as mpg  # noqa: E402  (plyfile's file format)
import mesh_types_cases as cases  # noqa: E402

mdg = mcg.mdg
import games.multi_mesh_splatting.scene.dataset_readers as multi_readers  # noqa: E402
import games.flame_splatting.scene.dataset_readers as flame_readers  # noqa: E402
from utils.camera_utils import cameraList_from_camInfos  # noqa: E402


class _Mesh(mdg._Mesh):
    def __init__(self, path):
        super().__init__(path)
        self.triangles = self.vertices[self.faces]


multi_readers.trimesh = types.SimpleNamespace(load=lambda path, force=None: _Mesh(path))
_EMBEDDING = os.path.join(tempfile.gettempdir(), "gms_static_embedding.pkl")


class _FlameConfig(flame_readers.FlameConfig):
    def __init__(self):
        super().__init__()
        self.flame_model_path = cases.FLAME_MODEL
        self.static_landmark_embedding_path = _EMBEDDING
        self.use_face_contour = False


flame_readers.FlameConfig = _FlameConfig

CFG_ARGV = {
    "multi": ["-s", "<SRC>", "-m", "<OUT>", "--gs_type", "gs_multi_mesh", "--meshes", "a", "b", "--num_splats", "2", "3",
              "--eval", "--iterations", "40"],
    "flame": ["-s", "<SRC>", "-m", "<OUT>", "--gs_type", "gs_flame", "-w", "--sh_degree", "2", "--flame_shape_lr", "0.02"],
}


def safe_state():
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)


def cameras(info, key, res):
    random.shuffle(info.train_cameras)
    random.shuffle(info.test_cameras)
    res[f"{key}/extent"] = np.array(info.nerf_normalization["radius"], np.float64)
    args = types.SimpleNamespace(resolution=-1, data_device="cpu")
    for split, infos in (("train", info.train_cameras), ("test", info.test_cameras)):
        cams = cameraList_from_camInfos(infos, 1.0, args)
        res[f"{key}/{split}/names"] = np.array([c.image_name for c in cams], dtype="U64")
        res[f"{key}/{split}/R"] = np.array([c.R for c in cams], np.float64).reshape(-1, 3, 3)
        res[f"{key}/{split}/T"] = np.array([c.T for c in cams], np.float64).reshape(-1, 3)
        res[f"{key}/{split}/fov"] = np.array([[c.FoVx, c.FoVy] for c in cams], np.float64).reshape(-1, 2)
        res[f"{key}/{split}/size"] = np.array([[c.image_width, c.image_height] for c in cams], np.int64).reshape(-1, 2)


def ply_bytes(rows, work) -> np.ndarray:
    path = os.path.join(work, "_cloud.ply")
    mpg.PlyData([mpg.PlyElement.describe(rows, "vertex")]).write(path)
    with open(path, "rb") as f:
        return np.frombuffer(f.read(), np.uint8).copy()


def main():
    import pickle
    with open(_EMBEDDING, "wb") as fh:
        pickle.dump(dict(lmk_face_idx=np.zeros(3, np.int64), lmk_b_coords=np.full((3, 3), 1 / 3)), fh, protocol=2)
    res = {}
    os.environ["OAR_JOB_ID"] = mcg.JOB_ID
    try:
        with tempfile.TemporaryDirectory() as d:
            src = {"multi": cases.write_multi(os.path.join(d, "multi")), "flame": cases.write_flame(os.path.join(d, "flame"))}
            mdg._PLY_FILES.clear()
            safe_state()
            info = multi_readers.readColmapMeshSceneInfo(src["multi"], "images", cases.MULTI_EVAL, cases.NUM_SPLATS, cases.MESHES)
            for i, p in enumerate(info.point_cloud):
                res[f"multi/mesh{i}/alpha"] = p.alpha.numpy().copy()
                res[f"multi/mesh{i}/colors"] = np.asarray(p.colors).copy()
                res[f"multi/mesh{i}/ply"] = ply_bytes(mdg._PLY_FILES[os.path.join(src["multi"], f"points3d_{i}.ply")], d)
            cameras(info, "multi", res)

            mdg._PLY_FILES.clear()
            safe_state()
            info = flame_readers.readNerfSyntheticFlameInfo(src["flame"], False, cases.FLAME_EVAL)
            p = info.point_cloud
            res["flame/alpha"] = p.alpha.numpy().copy()
            res["flame/colors"] = np.asarray(p.colors).copy()
            res["flame/vertices"] = p.vertices_init.detach().numpy().copy()
            res["flame/faces"] = p.faces.numpy().copy()
            rows = mdg._PLY_FILES[os.path.join(src["flame"], "points3d.ply")]
            for n in rows.dtype.names:
                res[f"flame/ply_{n}"] = np.ascontiguousarray(rows[n]).copy()
            cameras(info, "flame", res)

            for key, argv in CFG_ARGV.items():
                out = os.path.join(d, "cfg", key)
                os.makedirs(out)
                res[f"cfg/{key}/argv"] = np.array("\x1f".join(argv))
                res[f"cfg/{key}/text"] = np.array(mcg.reference_cfg_args(argv, src[key], out))
    finally:
        os.remove(_EMBEDDING)
    np.savez_compressed(os.path.join(HERE, "train_mesh_types.npz"), **res)
    print(f"{len(res)} arrays, {os.path.getsize(os.path.join(HERE, 'train_mesh_types.npz'))} bytes")


if __name__ == "__main__":
    main()
