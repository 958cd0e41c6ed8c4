"""Tiny scenes whose views differ in image size, written from fixed seeds on top of tests/dataset_cases.py, for the
mixed-size training tests (test_train_mixed_sizes_host.py, test_gpu_train_mixed_sizes.py):

  blender: a NeRF-synthetic scene with landscape and portrait PNGs (mesh.obj and points3d.ply included), the layout of a
           scene whose source images differ in size;
  colmap:  a COLMAP scene with two cameras of different sizes (a PINHOLE landscape sensor and a SIMPLE_PINHOLE portrait
           one), every camera looking at the origin, and the meshes a.obj / b.obj under sparse/0/ for gs_multi_mesh."""
from __future__ import annotations

import math
import os
import struct

import numpy as np

import dataset_cases
import mesh_types_cases
from gms_b200 import scenes

LANDSCAPE, PORTRAIT = (48, 32), (32, 48)
MESHES, NUM_SPLATS = ["a", "b"], [2, 3]


def write_blender(root: str, n_train: int = 6, n_test: int = 2, seed: int = 7) -> str:
    sizes = [LANDSCAPE, PORTRAIT]
    dataset_cases.write_blender(root, [sizes[i % 2] for i in range(n_train)], [sizes[i % 2] for i in range(n_test)], seed=seed,
                                mesh=True, points=True)
    return root


def colmap_cameras():
    """(camera id, model, (width, height), params) of the two sensors."""
    (W0, H0), (W1, H1) = LANDSCAPE, PORTRAIT
    f0, f1 = W0 / (2 * math.tan(0.4)), H1 / (2 * math.tan(0.45))
    return [(1, "PINHOLE", LANDSCAPE, [f0, f0 * 1.05, W0 / 2, H0 / 2]), (2, "SIMPLE_PINHOLE", PORTRAIT, [f1, W1 / 2, H1 / 2])]


def camera_of(k: int) -> int:
    """Index into colmap_cameras() of image k: alternating, shifted by one every eight images, so that both the --eval
    test views (every eighth) and the training views hold both sizes."""
    return (k + k // 8) % 2


def write_colmap(root: str, n_images: int = 16, seed: int = 8) -> str:
    """sparse/0/{cameras,images,points3D}.bin with the images spread over the two cameras (camera_of), RGB PNGs at each
    camera's size, 40 points, and two meshes a.obj / b.obj."""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    sparse = os.path.join(root, "sparse", "0")
    os.makedirs(sparse, exist_ok=True)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    cams = colmap_cameras()
    with open(os.path.join(sparse, "cameras.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(cams)))
        for cid, model, (W, H), p in cams:
            mid = {"SIMPLE_PINHOLE": 0, "PINHOLE": 1}[model]
            f.write(struct.pack("<iiQQ", cid, mid, W, H) + struct.pack("<" + "d" * len(p), *p))
    with open(os.path.join(sparse, "images.bin"), "wb") as f:
        f.write(struct.pack("<Q", n_images))
        for k in range(n_images):
            cid, _, (W, H), _ = cams[camera_of(k)]
            name = f"view_{k:02d}.png"
            dataset_cases.write_png(os.path.join(root, "images", name), rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
            c2w = dataset_cases._c2w(rng, radius=3.0)
            c2w[:3, 1:3] *= -1                              # Blender's camera axes to COLMAP's
            w2c = np.linalg.inv(c2w)
            x, y, z, w = Rotation.from_matrix(w2c[:3, :3]).as_quat()
            f.write(struct.pack("<idddddddi", k + 1, w, x, y, z, *w2c[:3, 3], cid) + name.encode() + b"\x00" + struct.pack("<Q", 0))
    xyz, rgb = rng.normal(size=(40, 3)) * 0.5, rng.integers(0, 256, (40, 3))
    with open(os.path.join(sparse, "points3D.bin"), "wb") as f:
        f.write(struct.pack("<Q", 40))
        for i in range(40):
            f.write(struct.pack("<QdddBBBd", i + 1, *xyz[i], *[int(c) for c in rgb[i]], 0.5) + struct.pack("<Q", 0))
    v, fc = scenes.icosphere(1, 0.6)
    mesh_types_cases.write_obj(os.path.join(sparse, "a.obj"), v, fc)
    v, fc = scenes.icosphere(0, 0.3)
    mesh_types_cases.write_obj(os.path.join(sparse, "b.obj"), v + np.array([0.4, -0.1, 0.2]), fc)
    return root
