"""The two scenes of the gs_multi_mesh / gs_flame reader fixture (tests/golden/make_train_mesh_types_golden.py,
tests/test_train_mesh_types_host.py), written from fixed seeds on top of tests/dataset_cases.py:

  multi: dataset_cases' COLMAP scene "colmap_bin" plus two OBJ meshes under sparse/0/ with different face counts, read
         with --meshes a b --num_splats 2 3 and --eval (llffhold 8);
  flame: dataset_cases' NeRF-synthetic scene "blender_a", trained with the FLAME model file
         tests/golden/flame_lbs/model_dense.pkl, without --eval (the test views join the training views)."""
from __future__ import annotations

import os

import numpy as np

import dataset_cases
from gms_b200 import scenes

HERE = os.path.dirname(os.path.abspath(__file__))
FLAME_MODEL = os.path.join(HERE, "golden", "flame_lbs", "model_dense.pkl")
MESHES, NUM_SPLATS = ["a", "b"], [2, 3]
MULTI_EVAL, FLAME_EVAL = True, False


def write_obj(path: str, verts: np.ndarray, faces: np.ndarray) -> None:
    with open(path, "w") as f:
        for x in verts:
            f.write("v %.6f %.6f %.6f\n" % tuple(x))
        for t in faces + 1:
            f.write("f %d %d %d\n" % tuple(t))


def write_multi(root: str) -> str:
    dataset_cases.DATASETS["colmap_bin"](root)
    rs = np.random.RandomState(11)
    v, f = scenes.icosphere(0, 0.7)
    write_obj(os.path.join(root, "sparse", "0", "a.obj"), v + 0.02 * rs.randn(*v.shape), f)
    v, f = scenes.icosphere(1, 0.4)
    write_obj(os.path.join(root, "sparse", "0", "b.obj"), v + np.array([0.5, -0.2, 0.1]) + 0.01 * rs.randn(*v.shape), f)
    return root


def write_flame(root: str) -> str:
    dataset_cases.DATASETS["blender_a"](root)
    return root
