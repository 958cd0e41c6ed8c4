"""Deterministic tiny datasets on disk for the loader tests (gms_b200/dataset.py) and their fixture
(tests/golden/make_dataset_golden.py).  Everything is generated from fixed seeds: PNGs through io_image.encode_png, COLMAP
sparse models through struct, a small mesh.obj.

CASES: name -> (writer, load_scene keyword arguments).  Together they cover alpha 0 / partial / 255 over white and black,
eval on and off, PINHOLE and SIMPLE_PINHOLE cameras in cameras.bin (PINHOLE in cameras.txt), names with two dots, and the
resolution rules: width 25 at -r 2 (12.5 rounds to 12), widths 1601 and 1617 at -r -1 (both become 1599), an explicit
-r 40, and -r 31 on 30-wide images (the width changes, the height does not)."""
from __future__ import annotations

import json
import math
import os
import struct

import numpy as np

from gms_b200 import io_image, io_ply, scenes


def write_png(path: str, arr: np.ndarray) -> None:
    H, W, Cn = arr.shape
    rows = np.concatenate([np.zeros((H, 1), np.uint8), arr.reshape(H, W * Cn)], axis=1)
    with open(path, "wb") as f:
        f.write(io_image.encode_png(rows.tobytes(), W, H, Cn))


def _rgba(rng, H, W):
    """Random colours; alpha 0, 255 or random per pixel, in about equal parts."""
    a = rng.integers(0, 256, (H, W), dtype=np.uint8)
    pick = rng.integers(0, 3, (H, W))
    a = np.where(pick == 0, 0, np.where(pick == 1, 255, a)).astype(np.uint8)
    return np.concatenate([rng.integers(0, 256, (H, W, 3), dtype=np.uint8), a[..., None]], axis=2)


def _c2w(rng, radius=4.0):
    """A Blender camera-to-world matrix looking at the origin from a random direction."""
    d = rng.normal(size=3)
    d /= np.linalg.norm(d)
    eye = d * radius
    back = d                                           # Blender cameras look down -z
    right = np.cross([0.0, 0.0, 1.0], back)
    right /= np.linalg.norm(right)
    up = np.cross(back, right)
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = right, up, back, eye
    return m


def write_blender(root: str, sizes_train, sizes_test, seed: int, mesh: bool = False, points: bool = False) -> None:
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "train"), exist_ok=True)
    os.makedirs(os.path.join(root, "test"), exist_ok=True)
    for split, sizes in (("train", sizes_train), ("test", sizes_test)):
        frames = []
        for i, (W, H) in enumerate(sizes):
            write_png(os.path.join(root, split, f"r_{i}.png"), _rgba(rng, H, W))
            frames.append({"file_path": f"./{split}/r_{i}", "transform_matrix": _c2w(rng).tolist()})
        with open(os.path.join(root, f"transforms_{split}.json"), "w") as f:
            json.dump({"camera_angle_x": scenes.NERF_FOVX, "frames": frames}, f)
    if mesh:
        v, fcs = scenes.icosphere(1, 0.8)
        with open(os.path.join(root, "mesh.obj"), "w") as f:
            for x in v:
                f.write("v %.6f %.6f %.6f\n" % tuple(x))
            for t in fcs + 1:
                f.write("f %d %d %d\n" % tuple(t))
    if points:
        io_ply.save_point_cloud(os.path.join(root, "points3d.ply"), rng.uniform(-1, 1, (50, 3)), rng.uniform(0, 255, (50, 3)))


def _qvec(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    return q if q[0] >= 0 else -q


def write_colmap(root: str, n_images: int, size, seed: int, text: bool = False, models=("PINHOLE", "SIMPLE_PINHOLE"),
                 rgba_image: bool = False) -> None:
    """sparse/0 with one camera per entry of `models` (images alternate between them), n_images RGB PNGs named
    `view_<k>.frame.png` (two dots) in shuffled order, and 40 points."""
    rng = np.random.default_rng(seed)
    sparse = os.path.join(root, "sparse", "0")
    os.makedirs(sparse, exist_ok=True)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    W, H = size
    ids = {"SIMPLE_PINHOLE": (0, 3), "PINHOLE": (1, 4), "OPENCV": (4, 8)}
    cams = []
    for cid, model in enumerate(models, 1):
        f = W / (2 * math.tan(0.35 + 0.05 * cid))
        params = {"SIMPLE_PINHOLE": [f, W / 2, H / 2], "PINHOLE": [f, f * 1.1, W / 2, H / 2],
                  "OPENCV": [f, f, W / 2, H / 2, 0.01, 0.0, 0.0, 0.0]}[model]
        cams.append((cid, model, params))
    order = rng.permutation(n_images)
    imgs = []
    for j, k in enumerate(order):
        name = f"view_{k:02d}.frame.png"
        arr = rng.integers(0, 256, (H, W, 4 if (rgba_image and j == 0) else 3), dtype=np.uint8)
        write_png(os.path.join(root, "images", name), arr)
        q, t = _qvec(rng), rng.normal(size=3) * 2
        imgs.append((j + 1, q, t, cams[j % len(cams)][0], name))
    xyz = rng.normal(size=(40, 3))
    rgb = rng.integers(0, 256, (40, 3))
    if text:
        with open(os.path.join(sparse, "cameras.txt"), "w") as f:
            f.write("# Camera list\n")
            for cid, model, p in cams:
                f.write(f"{cid} {model} {W} {H} " + " ".join(repr(float(x)) for x in p) + "\n")
        with open(os.path.join(sparse, "images.txt"), "w") as f:
            f.write("# Image list\n")
            for iid, q, t, cid, name in imgs:
                f.write(f"{iid} " + " ".join(repr(float(x)) for x in list(q) + list(t)) + f" {cid} {name}\n")
                f.write("1.5 2.5 -1 3.5 4.5 7\n")
        with open(os.path.join(sparse, "points3D.txt"), "w") as f:
            f.write("# 3D point list\n")
            for i in range(40):
                f.write(f"{i + 1} " + " ".join(repr(float(x)) for x in xyz[i]) + " " + " ".join(str(int(c)) for c in rgb[i])
                        + " 0.5 1 0 2 1\n")
        return
    with open(os.path.join(sparse, "cameras.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(cams)))
        for cid, model, p in cams:
            mid, npar = ids[model]
            f.write(struct.pack("<iiQQ", cid, mid, W, H) + struct.pack("<" + "d" * npar, *p))
    with open(os.path.join(sparse, "images.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(imgs)))
        for iid, q, t, cid, name in imgs:
            f.write(struct.pack("<idddddddi", iid, *q, *t, cid) + name.encode() + b"\x00")
            f.write(struct.pack("<Q", 2) + struct.pack("<ddqddq", 1.5, 2.5, -1, 3.5, 4.5, 7))
    with open(os.path.join(sparse, "points3D.bin"), "wb") as f:
        f.write(struct.pack("<Q", 40))
        for i in range(40):
            f.write(struct.pack("<QdddBBBd", i + 1, *xyz[i], *[int(c) for c in rgb[i]], 0.5))
            f.write(struct.pack("<Q", 2) + struct.pack("<iiii", 1, 0, 2, 1))


DATASETS = {
    "blender_a": lambda r: write_blender(r, [(25, 17)] * 3, [(25, 17)] * 2, seed=1, mesh=True),
    "blender_wide": lambda r: write_blender(r, [(1601, 9), (1617, 11)], [(30, 20)], seed=2, points=True),
    "colmap_bin": lambda r: write_colmap(r, 9, (50, 36), seed=3),
    "colmap_txt": lambda r: write_colmap(r, 9, (30, 20), seed=4, text=True, models=("PINHOLE",)),
    "colmap_opencv": lambda r: write_colmap(r, 2, (20, 10), seed=5, models=("OPENCV",)),
    "colmap_rgba": lambda r: write_colmap(r, 2, (20, 10), seed=6, rgba_image=True),
}

# fixture cases: (dataset, load_scene keyword arguments)
CASES = {
    "blender_white_r2": ("blender_a", dict(gs_type="gs", white_background=True, eval=False, resolution=2)),
    "blender_mesh_eval": ("blender_a", dict(gs_type="gs_mesh", white_background=False, eval=True, resolution=-1, num_splats=2)),
    "blender_wide": ("blender_wide", dict(gs_type="gs_flat", white_background=False, eval=False, resolution=-1)),
    "colmap_bin_eval_r40": ("colmap_bin", dict(gs_type="gs", eval=True, resolution=40)),
    "colmap_txt_r31": ("colmap_txt", dict(gs_type="gs_flat", eval=False, resolution=31)),
}


def write_all(root: str) -> dict:
    """Writes every dataset under root; -> {dataset name: its directory}."""
    out = {}
    for name, fn in DATASETS.items():
        d = os.path.join(root, name)
        fn(d)
        out[name] = d
    return out
