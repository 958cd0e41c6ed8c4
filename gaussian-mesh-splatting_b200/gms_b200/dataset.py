"""Datasets on disk -> the cameras and 8-bit ground-truth images the native trainers and renderers consume.

Restates the reference's scene loading (no reference code is imported):
  * NeRF-synthetic: readCamerasFromTransforms / readNerfSyntheticInfo   scene/dataset_readers.py:179-258
  * COLMAP: readColmapSceneInfo / readColmapCameras                      scene/dataset_readers.py:68-105, 132-177
    and the sparse-model readers                                         scene/colmap_loader.py
  * gs_mesh scenes: readNerfSyntheticMeshInfo                            games/mesh_splatting/scene/dataset_readers.py:40-105
    with GaussianMeshModel.create_from_pcd                               games/mesh_splatting/scene/gaussian_mesh_model.py:49-84
  * gs_multi_mesh scenes: readColmapMeshSceneInfo                        games/multi_mesh_splatting/scene/dataset_readers.py:38-114
    with GaussianMultiMeshModel.create_from_pcd                          games/multi_mesh_splatting/scene/gaussian_multi_mesh_model.py:35-77
  * gs_flame scenes: readNerfSyntheticFlameInfo                          games/flame_splatting/scene/dataset_readers.py:48-130
  * resolution: loadCam                                                  utils/camera_utils.py:19-52
  * cameras_extent: getNerfppNorm                                        scene/dataset_readers.py:45-66
  * the shuffle and the training loop's view order                       scene/__init__.py:84-86, train.py:90-92

Images are decoded on the host (PIL when importable, else io_image.decode_png for PNG), staged through pinned memory and
prepared on the GPU: gms_image_composite_rgba puts Blender's RGBA over the background exactly as the reference's numpy does,
gms_image_resize_u8 is PILtoTorch's Image.resize bit for bit.  Every view stays resident as uint8 [H,W,3] (a quarter of the
float32 [3,H,W] the reference keeps); the trainers dequantize it per step.

Unlike the reference, nothing is written into the source directory: the reference stores points3d.ply / points3D.ply (and
points3d_<i>.ply for gs_multi_mesh) there and reads it back; here the same float32 / byte round trip
(io_ply.point_cloud_elements -> point_cloud_arrays) happens in memory, and the clouds a gs_mesh, gs_multi_mesh or gs_flame
run stores as its input ply are rebuilt from the initial parameters (mesh_input_cloud, Scene.mesh_clouds, flame_input_cloud).
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os
import random
import struct
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field
from pathlib import Path
from typing import List, Optional, Tuple

import numpy as np
import torch

from . import _lib, io_image, io_obj, io_ply, scenes
from .scenes import SH_C0, ZFAR, ZNEAR, Camera, MeshGaussianParams

# ------------------------------------------------------------------------------------------------ Pillow's resample tables

RESAMPLE_BITS = 22      # Pillow's PRECISION_BITS for 8-bit images


def _bicubic(x: np.ndarray) -> np.ndarray:
    """Pillow's bicubic_filter, a = -0.5, in the same operation order."""
    x = np.abs(x)
    near = ((1.5 * x - 2.5) * x) * x + 1.0
    far = ((((x - 5.0) * x) + 8.0) * x - 4.0) * -0.5
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def resize_coeffs(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray]:
    """One axis of Pillow's BICUBIC resample, precompute_coeffs + normalize_coeffs_8bpc: (bounds int32 [out,2] = (first
    source index, taps), coeffs int32 [out,ksize]).  support = 2 * max(scale, 1), center = (i + 0.5) * scale, xmin =
    int(center - support + 0.5); the weights are divided by their sum accumulated left to right, then rounded as
    int(+-0.5 + w * 2^22)."""
    if in_size < 1 or out_size < 1:
        raise ValueError(f"resize_coeffs: sizes must be >= 1; got {in_size} -> {out_size}")
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    xmin = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    xmax = np.minimum(np.trunc(center + support + 0.5).astype(np.int64), in_size)
    n = xmax - xmin
    t = np.arange(ksize)
    w = _bicubic(((t[None, :] + xmin[:, None]).astype(np.float64) - center[:, None] + 0.5) * (1.0 / filterscale))
    w = np.where(t[None, :] < n[:, None], w, 0.0)
    ww = np.zeros(out_size)
    for j in range(ksize):          # left to right, as Pillow's loop (numpy's pairwise sum would round differently)
        ww = ww + w[:, j]
    k = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    fixed = np.where(k < 0, np.trunc(-0.5 + k * float(1 << RESAMPLE_BITS)), np.trunc(0.5 + k * float(1 << RESAMPLE_BITS)))
    return np.stack([xmin, n], 1).astype(np.int32), fixed.astype(np.int32)


def camera_resolution(orig_w: int, orig_h: int, resolution: int = -1) -> Tuple[int, int]:
    """loadCam's (width, height) at resolution_scale 1: -r 1/2/4/8 divides with Python's round (halves to even); -1 scales
    images wider than 1600 to int(orig_w / (orig_w / 1600)) -- 1599 for some widths, e.g. 1601; any other value is a target
    width, both sides truncated."""
    if resolution in (1, 2, 4, 8):
        w, h = round(orig_w / resolution), round(orig_h / resolution)
    else:
        if resolution == -1:
            down = orig_w / 1600 if orig_w > 1600 else 1
        else:
            down = orig_w / resolution
        scale = float(down) * 1.0
        w, h = int(orig_w / scale), int(orig_h / scale)
    if w < 1 or h < 1:
        raise ValueError(f"resolution {resolution} turns a {orig_w}x{orig_h} image into {w}x{h}")
    return w, h


# ------------------------------------------------------------------------------------------------ cameras

def fov2focal(fov: float, pixels: int) -> float:
    return pixels / (2 * math.tan(fov / 2))


def focal2fov(focal: float, pixels: int) -> float:
    return 2 * math.atan(pixels / (2 * focal))


def world_to_view(R: np.ndarray, T: np.ndarray) -> np.ndarray:
    """getWorld2View2 (utils/graphics_utils.py:38-49) with zero translate and unit scale, the same two inversions, float32."""
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = R.transpose()
    Rt[:3, 3] = T
    Rt[3, 3] = 1.0
    C2W = np.linalg.inv(Rt)
    C2W[:3, 3] = (C2W[:3, 3] + np.array([0.0, 0.0, 0.0])) * 1.0
    return np.float32(np.linalg.inv(C2W))


def make_camera(R, T, fovx: float, fovy: float, width: int, height: int, uid) -> Camera:
    """scene/cameras.py:54-57: transposed float32 world->view, projection, their product and the camera centre."""
    wvt = torch.tensor(world_to_view(R, T)).transpose(0, 1)
    proj = scenes.projection_matrix(ZNEAR, ZFAR, fovx, fovy).transpose(0, 1)
    full = wvt.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0)
    center = wvt.inverse()[3, :3]
    return Camera(int(width), int(height), fovx, fovy, wvt.contiguous(), full.contiguous(), center.contiguous(), uid)


def nerfpp_radius(infos) -> float:
    """getNerfppNorm's radius: 1.1 x the largest distance of a camera centre (inverse of the float32 world->view) from
    their mean, in numpy's dtypes."""
    centers = [np.linalg.inv(world_to_view(i.R, i.T))[:3, 3:4] for i in infos]
    cc = np.hstack(centers)
    dist = np.linalg.norm(cc - np.mean(cc, axis=1, keepdims=True), axis=0, keepdims=True)
    return float(np.max(dist) * 1.1)


@dataclass
class ViewInfo:
    """CameraInfo (scene/dataset_readers.py:26-36) without the image: R (transposed W2C rotation), T, FoVs, the file."""
    R: np.ndarray
    T: np.ndarray
    FovX: float
    FovY: float
    path: str
    name: str
    width: int = 0
    height: int = 0


# ------------------------------------------------------------------------------------------------ NeRF-synthetic

def read_transforms(path: str, transformsfile: str, extension: str = ".png") -> List[ViewInfo]:
    """readCamerasFromTransforms' cameras: c2w[:3,1:3] *= -1, R = inv(c2w)[:3,:3]^T, T = inv(c2w)[:3,3]; the name is the
    file's stem.  FovY needs the image's size; read_scene fills it in."""
    with open(os.path.join(path, transformsfile)) as f:
        contents = json.load(f)
    fovx = contents["camera_angle_x"]
    out = []
    for frame in contents["frames"]:
        cam_name = os.path.join(path, frame["file_path"][2:] + extension)
        c2w = np.array(frame["transform_matrix"])
        c2w[:3, 1:3] *= -1
        w2c = np.linalg.inv(c2w)
        out.append(ViewInfo(np.transpose(w2c[:3, :3]), w2c[:3, 3], fovx, 0.0, cam_name, Path(cam_name).stem))
    return out


# ------------------------------------------------------------------------------------------------ COLMAP

# COLMAP's camera models: id -> (name, number of parameters).  Only the undistorted ones are loaded.
COLMAP_MODELS = {0: ("SIMPLE_PINHOLE", 3), 1: ("PINHOLE", 4), 2: ("SIMPLE_RADIAL", 4), 3: ("RADIAL", 5), 4: ("OPENCV", 8),
                 5: ("OPENCV_FISHEYE", 8), 6: ("FULL_OPENCV", 12), 7: ("FOV", 5), 8: ("SIMPLE_RADIAL_FISHEYE", 4),
                 9: ("RADIAL_FISHEYE", 5), 10: ("THIN_PRISM_FISHEYE", 12)}


def _unpack(f, fmt: str):
    fmt = "<" + fmt
    data = f.read(struct.calcsize(fmt))
    return struct.unpack(fmt, data)


def read_colmap_cameras(sparse: str) -> dict:
    """cameras.bin, else cameras.txt -> {camera_id: (model name, width, height, params float64)}."""
    cams = {}
    try:
        with open(os.path.join(sparse, "cameras.bin"), "rb") as f:
            for _ in range(_unpack(f, "Q")[0]):
                cid, model_id, w, h = _unpack(f, "iiQQ")
                if model_id not in COLMAP_MODELS:
                    raise ValueError(f"{sparse}/cameras.bin: unknown COLMAP camera model id {model_id}")
                name, npar = COLMAP_MODELS[model_id]
                cams[cid] = (name, int(w), int(h), np.array(_unpack(f, "d" * npar)))
        return cams
    except FileNotFoundError:
        pass
    with open(os.path.join(sparse, "cameras.txt")) as f:
        for line in f:
            line = line.strip()
            if line and line[0] != "#":
                e = line.split()
                cams[int(e[0])] = (e[1], int(e[2]), int(e[3]), np.array(tuple(map(float, e[4:]))))
    return cams


def read_colmap_images(sparse: str) -> list:
    """images.bin, else images.txt -> [(qvec, tvec, camera_id, name)] in file order."""
    out = []
    try:
        with open(os.path.join(sparse, "images.bin"), "rb") as f:
            for _ in range(_unpack(f, "Q")[0]):
                p = _unpack(f, "idddddddi")
                name = b""
                while (ch := f.read(1)) != b"\x00":
                    if not ch:
                        raise ValueError(f"{sparse}/images.bin: truncated image name")
                    name += ch
                n2d = _unpack(f, "Q")[0]
                f.seek(24 * n2d, 1)
                out.append((np.array(p[1:5]), np.array(p[5:8]), p[8], name.decode("utf-8")))
        return out
    except FileNotFoundError:
        pass
    with open(os.path.join(sparse, "images.txt")) as f:
        lines = iter(f)
        for line in lines:
            line = line.strip()
            if line and line[0] != "#":
                e = line.split()
                out.append((np.array(tuple(map(float, e[1:5]))), np.array(tuple(map(float, e[5:8]))), int(e[8]), e[9]))
                next(lines, None)       # the 2D points line
    return out


def read_colmap_points(sparse: str) -> Tuple[np.ndarray, np.ndarray]:
    """points3D.bin, else points3D.txt -> (xyz float64 [P,3], rgb float64 [P,3])."""
    try:
        with open(os.path.join(sparse, "points3D.bin"), "rb") as f:
            n = _unpack(f, "Q")[0]
            xyz, rgb = np.empty((n, 3)), np.empty((n, 3))
            for i in range(n):
                p = _unpack(f, "QdddBBBd")
                xyz[i], rgb[i] = p[1:4], p[4:7]
                f.seek(8 * _unpack(f, "Q")[0], 1)
            return xyz, rgb
    except FileNotFoundError:
        pass
    xyz, rgb = [], []
    with open(os.path.join(sparse, "points3D.txt")) as f:
        for line in f:
            line = line.strip()
            if line and line[0] != "#":
                e = line.split()
                xyz.append(tuple(map(float, e[1:4])))
                rgb.append(tuple(map(int, e[4:7])))
    return np.array(xyz, np.float64).reshape(-1, 3), np.array(rgb, np.float64).reshape(-1, 3)


def qvec2rotmat(q) -> np.ndarray:
    """COLMAP's (w, x, y, z) quaternion -> rotation matrix, in colmap_loader's operation order."""
    return np.array([
        [1 - 2 * q[2] ** 2 - 2 * q[3] ** 2, 2 * q[1] * q[2] - 2 * q[0] * q[3], 2 * q[3] * q[1] + 2 * q[0] * q[2]],
        [2 * q[1] * q[2] + 2 * q[0] * q[3], 1 - 2 * q[1] ** 2 - 2 * q[3] ** 2, 2 * q[2] * q[3] - 2 * q[0] * q[1]],
        [2 * q[3] * q[1] - 2 * q[0] * q[2], 2 * q[2] * q[3] + 2 * q[0] * q[1], 1 - 2 * q[1] ** 2 - 2 * q[2] ** 2]])


def read_colmap(path: str, images: str = "images") -> List[ViewInfo]:
    """readColmapCameras + the sort by name: R = qvec2rotmat(q)^T, T = t; FoVs from the focal lengths of PINHOLE (fx, fy)
    or SIMPLE_PINHOLE (f) cameras; the name is the basename up to its first dot."""
    sparse = os.path.join(path, "sparse/0")
    cams = read_colmap_cameras(sparse)
    folder = os.path.join(path, images)
    out = []
    for q, t, cid, name in read_colmap_images(sparse):
        model, w, h, params = cams[cid]
        if model == "SIMPLE_PINHOLE":
            fx = fy = params[0]
        elif model == "PINHOLE":
            fx, fy = params[0], params[1]
        else:
            raise ValueError(f"COLMAP camera model {model} is not supported: only undistorted datasets (PINHOLE or "
                             f"SIMPLE_PINHOLE cameras) can be loaded")
        image_path = os.path.join(folder, os.path.basename(name))
        out.append(ViewInfo(np.transpose(qvec2rotmat(q)), np.array(t), focal2fov(fx, w), focal2fov(fy, h), image_path,
                            os.path.basename(image_path).split(".")[0], w, h))
    return sorted(out, key=lambda v: v.name)


# ------------------------------------------------------------------------------------------------ image decode (host)

def image_size(path: str) -> Tuple[int, int]:
    """(width, height) from the file's header: PIL when importable, else PNG's IHDR."""
    try:
        from PIL import Image
    except ImportError:
        Image = None
    if Image is not None:
        with Image.open(path) as im:
            return im.size
    with open(path, "rb") as f:
        head = f.read(24)
    if head[:8] != b"\x89PNG\r\n\x1a\n":
        raise RuntimeError(f"{path}: only PNG images can be read without Pillow")
    return struct.unpack(">II", head[16:24])


def decode_image(path: str, mode: str) -> np.ndarray:
    """-> uint8 [H,W,4] for mode "RGBA" (convert("RGBA")), uint8 [H,W,3] for "RGB" (the file must be RGB).  PIL when
    importable; otherwise PNG only, grey / RGB expanded to RGBA as convert("RGBA") does."""
    try:
        from PIL import Image
    except ImportError:
        Image = None
    if Image is not None:
        with Image.open(path) as im:
            if mode == "RGBA":
                return np.asarray(im.convert("RGBA"))
            if im.mode != "RGB":
                raise ValueError(f"{path}: image mode {im.mode!r}; COLMAP ground truth must be RGB")
            return np.asarray(im)
    with open(path, "rb") as f:
        data = f.read()
    if data[:8] != b"\x89PNG\r\n\x1a\n":
        raise RuntimeError(f"{path}: only PNG images can be decoded without Pillow")
    arr = io_image.decode_png(data)
    ch = arr.shape[2]
    if mode == "RGB":
        if ch != 3:
            raise ValueError(f"{path}: image mode {({1: 'L', 4: 'RGBA'})[ch]!r}; COLMAP ground truth must be RGB")
        return arr
    if ch == 4:
        return arr
    rgb = np.repeat(arr, 3, axis=2) if ch == 1 else arr
    return np.concatenate([rgb, np.full(rgb.shape[:2] + (1,), 255, np.uint8)], axis=2)


# ------------------------------------------------------------------------------------------------ GPU preparation

class GroundTruthPreparer:
    """Host bytes -> resident uint8 [H,W,3] device images: pinned staging (two slots, reused once their copy is done),
    gms_image_composite_rgba for RGBA, gms_image_resize_u8 when the size changes.  Everything runs on the current stream."""

    def __init__(self, device="cuda"):
        self.dev = torch.device(device)
        self._stage = [None, None]
        self._events = [None, None]
        self._slot = 0
        self._tables = {}

    def _table(self, n_in: int, n_out: int):
        key = (n_in, n_out)
        if key not in self._tables:
            b, k = resize_coeffs(n_in, n_out)
            self._tables[key] = (torch.from_numpy(b).to(self.dev), torch.from_numpy(k).to(self.dev), k.shape[1], b)
        return self._tables[key]

    def upload(self, arr: np.ndarray) -> torch.Tensor:
        """uint8 host array -> device tensor of the same shape, through a pinned slot."""
        s = self._slot
        self._slot ^= 1
        if self._events[s] is not None:
            self._events[s].synchronize()       # the slot's previous copy has left the pinned buffer
        n = arr.size
        if self._stage[s] is None or self._stage[s].numel() < n:
            self._stage[s] = torch.empty(n, dtype=torch.uint8).pin_memory()
        stage = self._stage[s][:n]
        stage.numpy()[:] = np.ascontiguousarray(arr).reshape(-1)
        out = torch.empty(arr.shape, dtype=torch.uint8, device=self.dev)
        out.view(-1).copy_(stage, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.dev))
        self._events[s] = ev
        return out

    def composite(self, rgba: torch.Tensor, white_background: bool) -> torch.Tensor:
        H, W, _ = rgba.shape
        out = torch.empty(H, W, 3, dtype=torch.uint8, device=self.dev)
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().gms_image_composite_rgba(rgba.data_ptr(), out.data_ptr(), H, W, int(bool(white_background)),
                                                          torch.cuda.current_stream(self.dev).cuda_stream), "gms_image_composite_rgba")
        return out

    def resize(self, rgb: torch.Tensor, width: int, height: int) -> torch.Tensor:
        """uint8 [H,W,3] device -> [height,width,3], Image.resize's default filter."""
        H, W, _ = rgb.shape
        if (W, H) == (width, height):
            return rgb
        a = _lib.ResizeArgs()
        a.in_w, a.in_h, a.out_w, a.out_h, a.C = W, H, width, height, 3
        out = torch.empty(height, width, 3, dtype=torch.uint8, device=self.dev)
        a.src, a.dst = rgb.data_ptr(), out.data_ptr()
        scratch = None
        if W != width:
            bh, kh, a.ksize_h, _ = self._table(W, width)
            a.bounds_h, a.coeffs_h = bh.data_ptr(), kh.data_ptr()
        if H != height:
            bv, kv, a.ksize_v, bv_host = self._table(H, height)
            a.bounds_v, a.coeffs_v = bv.data_ptr(), kv.data_ptr()
            a.row0 = int(bv_host[0, 0])
            a.rows = int(bv_host[-1, 0] + bv_host[-1, 1]) - a.row0
            if W != width:
                scratch = torch.empty(width * a.rows * 3, dtype=torch.uint8, device=self.dev)
                a.scratch, a.scratch_bytes = scratch.data_ptr(), scratch.numel()
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().gms_image_resize_u8(C.byref(a), torch.cuda.current_stream(self.dev).cuda_stream),
                       "gms_image_resize_u8")
        return out


def _decoded(paths, mode: str, workers: int):
    """decode_image over `paths` in order, a few images ahead on a thread pool (the result does not depend on it)."""
    if workers <= 1:
        for p in paths:
            yield decode_image(p, mode)
        return
    with ThreadPoolExecutor(workers) as ex:
        pending = []
        for p in paths:
            pending.append(ex.submit(decode_image, p, mode))
            if len(pending) > 2 * workers:
                yield pending.pop(0).result()
        for f in pending:
            yield f.result()


# ------------------------------------------------------------------------------------------------ scenes

@dataclass
class Scene:
    """A loaded dataset.  Camera uid = the view's index in its (shuffled) list, loadCam's `id`."""
    train_cameras: List[Camera]
    test_cameras: List[Camera]
    train_views: List[ViewInfo]
    test_views: List[ViewInfo]
    cameras_extent: float
    point_cloud: Optional[Tuple[np.ndarray, np.ndarray, np.ndarray]] = None    # (points, colors, normals) as fetchPly
    mesh: Optional[MeshGaussianParams] = None                                   # gs_mesh initial parameters
    meshes: Optional[List[MeshGaussianParams]] = None                           # gs_multi_mesh: per mesh, in --meshes order
    mesh_clouds: Optional[List[Tuple[np.ndarray, np.ndarray]]] = None           # gs_multi_mesh: per mesh, points3d_<i>.ply's cloud
    flame: Optional["FlameInit"] = None                                         # gs_flame
    train_images: List[torch.Tensor] = field(default_factory=list)            # resident uint8 [H,W,3] (load_scene)
    test_images: List[torch.Tensor] = field(default_factory=list)
    mode: str = "RGB"                   # what the files decode to: "RGBA" (NeRF-synthetic, composited) or "RGB" (COLMAP)
    white_background: bool = False
    _rng_state: object = field(default=None, repr=False)

    @property
    def train_names(self) -> List[str]:
        return [v.name for v in self.train_views]

    @property
    def test_names(self) -> List[str]:
        return [v.name for v in self.test_views]

    def view_order(self, n: int) -> List[int]:
        """The training views the reference's first n iterations visit: the Random stream that shuffled the views goes on
        with viewpoint_stack.pop(randint(0, len - 1)), the stack refilled with every training view when empty."""
        rng = random.Random()
        rng.setstate(self._rng_state)
        order, stack = [], []
        for _ in range(n):
            if not stack:
                stack = list(range(len(self.train_cameras)))
            order.append(stack.pop(rng.randint(0, len(stack) - 1)))
        return order


def transform_vertices(vertices: torch.Tensor) -> torch.Tensor:
    """transform_vertices_function (games/mesh_splatting/scene/dataset_readers.py:33-37): swap y and z, negate the new y."""
    v = vertices[:, [0, 2, 1]]
    v[:, 1] = -v[:, 1]
    return v


def mesh_gaussians_from_obj(obj_path: str, num_splats: int, seed: int = 0) -> MeshGaussianParams:
    """readNerfSyntheticMeshInfo + GaussianMeshModel.create_from_pcd: the mesh through transform_vertices; alpha =
    torch.rand(F, K, 3) of a CPU generator seeded `seed`; colours SH2RGB(RandomState(seed).random_sample((F*K, 3)) / 255)
    (not truncated to bytes: the reference trains from the in-memory cloud), DC = RGB2SH of them in float32, rest 0,
    _scale = 1, opacity = inverse_sigmoid(0.1).

    io_obj.read_obj keeps the file's vertices as written; trimesh's default processing (which the reference loads through)
    merges duplicate vertices first, so a file with duplicates yields more vertices here."""
    verts, faces = io_obj.read_obj(obj_path)
    vertices = transform_vertices(verts)
    F, K = faces.shape[0], int(num_splats)
    P = F * K
    alpha = torch.rand(F, K, 3, generator=torch.Generator().manual_seed(seed))
    shs = np.random.RandomState(seed).random_sample((P, 3)) / 255.0
    colors = shs * SH_C0 + 0.5
    fdc = ((torch.tensor(colors).float() - 0.5) / SH_C0).reshape(P, 1, 3).contiguous()
    x = 0.1 * torch.ones(P, 1)
    opacity = torch.log(x / (1 - x))
    return MeshGaussianParams(vertices.contiguous(), faces, alpha, torch.ones(P, 1), fdc, torch.zeros(P, 15, 3), opacity)


def mesh_input_cloud(mesh: MeshGaussianParams, seed: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """The cloud readNerfSyntheticMeshInfo stores (storePly, the `input.ply` of a gs_mesh run) for mesh_gaussians_from_obj's
    parameters: points = torch.rand alpha (not normalised) @ the face's float32 triangle, colours SH2RGB(shs) * 255 in float64
    (save_point_cloud truncates them to bytes).  -> (points float32 [F*K,3], colours float64 [F*K,3])."""
    alpha = mesh._alpha.detach().cpu()
    F, K = alpha.shape[0], alpha.shape[1]
    triangles = mesh.vertices.detach().cpu()[mesh.faces.detach().cpu().long()].float()
    xyz = torch.matmul(alpha, triangles).reshape(F * K, 3)
    shs = np.random.RandomState(seed).random_sample((F * K, 3)) / 255.0
    return xyz.numpy(), (shs * SH_C0 + 0.5) * 255


def mesh_draws(F: int, K: int, gen: torch.Generator, rs: np.random.RandomState) -> Tuple[torch.Tensor, np.ndarray]:
    """One mesh's random initialisation in the reference readers' order: alpha = torch.rand(F, K, 3) from `gen`, then
    shs = random((F*K, 3)) / 255 from `rs` (float64)."""
    alpha = torch.rand(F, int(K), 3, generator=gen)
    shs = rs.random_sample((F * int(K), 3)) / 255.0
    return alpha, shs


def multi_mesh_gaussians(source_path: str, meshes: List[str], num_splats: List[int], seed: int = 0):
    """readColmapMeshSceneInfo + GaussianMultiMeshModel.create_from_pcd: mesh i is sparse/0/<meshes[i]>.obj as written (no
    transform_vertices), its alpha and colours drawn mesh by mesh from one torch CPU generator and one RandomState, both
    seeded `seed` (the reference's global streams after safe_state); DC = RGB2SH of SH2RGB(shs) in float32, rest 0, _scale 1,
    opacity inverse_sigmoid(0.1).  -> (per-mesh MeshGaussianParams, per-mesh (points float32 [F*K,3], colours float64
    [F*K,3]): the cloud storePly writes as points3d_<i>.ply, alpha @ the float32 triangles and SH2RGB(shs) * 255)."""
    if len(meshes) != len(num_splats):
        raise ValueError(f"gs_multi_mesh needs one --num_splats per --meshes entry; got {len(num_splats)} for {len(meshes)} meshes")
    gen, rs = torch.Generator().manual_seed(int(seed)), np.random.RandomState(seed)
    params, clouds = [], []
    for name, K in zip(meshes, num_splats):
        verts, faces = io_obj.read_obj(os.path.join(source_path, "sparse", "0", f"{name}.obj"))
        F, P = faces.shape[0], faces.shape[0] * int(K)
        alpha, shs = mesh_draws(F, K, gen, rs)
        triangles = verts[faces]
        clouds.append((torch.matmul(alpha, triangles).reshape(P, 3).numpy(), (shs * SH_C0 + 0.5) * 255))
        fdc = ((torch.tensor(shs * SH_C0 + 0.5).float() - 0.5) / SH_C0).reshape(P, 1, 3).contiguous()
        x = 0.1 * torch.ones(P, 1)
        params.append(MeshGaussianParams(verts.contiguous(), faces, alpha, torch.ones(P, 1), fdc, torch.zeros(P, 15, 3),
                                         torch.log(x / (1 - x))))
    return params, clouds


FLAME_K = 100       # readNerfSyntheticFlameInfo's num_pts_each_triangle
DEFAULT_FLAME_MODEL = os.path.join("games", "flame_splatting", "FLAME", "model", "flame2023.pkl")   # FlameConfig's path


@dataclass
class FlameInit:
    """What readNerfSyntheticFlameInfo draws on the host: the FLAME model file, its faces (int64 [F,3]), alpha =
    torch.rand(F, 100, 3) and SH2RGB(shs) (float64 [F*100,3]) from generators seeded `seed` -- the draws
    FlameGaussianModel.create(driver, faces, K=100, seed=seed) makes.  The mesh itself needs the driver
    (flame_input_cloud)."""
    model_path: str
    faces: torch.Tensor
    alpha: torch.Tensor
    colors: np.ndarray
    seed: int = 0


def flame_init(model_path: str, seed: int = 0) -> FlameInit:
    from . import flame as _flame
    faces = torch.tensor(np.asarray(_flame.read_model_file(model_path)["f"]).astype(np.int64))
    alpha, shs = mesh_draws(faces.shape[0], FLAME_K, torch.Generator().manual_seed(int(seed)), np.random.RandomState(seed))
    return FlameInit(model_path, faces, alpha, shs * SH_C0 + 0.5, int(seed))


def flame_input_cloud(model, init: FlameInit) -> Tuple[np.ndarray, np.ndarray]:
    """readNerfSyntheticFlameInfo's points3d.ply (the `input.ply` of a gs_flame run) for the FlameGaussianModel built from
    `init`: alpha (the raw torch.rand draws, not the softmax) @ the triangles of the mesh at the model's current parameters
    (zero and enlargement 8.35 for a new model), colours SH2RGB(shs) * 255 (float64; save_point_cloud truncates them to
    bytes).  -> (points float32 [F*K,3], colours float64 [F*K,3])."""
    verts = model.refresh_vertices().detach()
    alpha = model._alpha.detach()
    F, K = alpha.shape[0], alpha.shape[1]
    xyz = torch.matmul(alpha, verts[model.faces]).reshape(F * K, 3)
    return xyz.cpu().numpy(), init.colors * 255


SUPPORTED = {"blender": ("gs", "gs_flat", "gs_mesh", "gs_flame"), "colmap": ("gs", "gs_flat", "gs_multi_mesh")}


def read_scene(source_path: str, gs_type: str, white_background: bool = False, eval: bool = False, resolution: int = -1,
               images: str = "images", num_splats=2, seed: int = 0, shuffle: bool = True, meshes: Optional[List[str]] = None,
               flame_model: str = DEFAULT_FLAME_MODEL) -> Scene:
    """Everything of load_scene but the images, on the host: cameras (CPU tensors), names, extent, point cloud or mesh
    parameters and the view-order stream.  Image files are only opened for their size.

    num_splats: K of a gs_mesh scene (an int), or a list with one K per entry of `meshes` for gs_multi_mesh.  flame_model:
    the FLAME model file of a gs_flame scene (the reference's default path, relative to the working directory)."""
    if os.path.exists(os.path.join(source_path, "sparse")):
        kind = "colmap"
    elif os.path.exists(os.path.join(source_path, "transforms_train.json")):
        kind = "blender"
    else:
        raise ValueError(f"{source_path}: neither a COLMAP (sparse/) nor a NeRF-synthetic (transforms_train.json) scene")
    if gs_type not in SUPPORTED[kind]:
        raise ValueError(f"gs_type {gs_type!r} is not supported on {kind} scenes (supported: {', '.join(SUPPORTED[kind])})")
    if kind == "blender":
        train = read_transforms(source_path, "transforms_train.json")
        test = read_transforms(source_path, "transforms_test.json")
        for v in train + test:
            v.width, v.height = image_size(v.path)
            v.FovY = focal2fov(fov2focal(v.FovX, v.width), v.height)
        if not eval:
            train, test = train + test, []
    else:
        views = read_colmap(source_path, images)
        if eval:
            train = [v for i, v in enumerate(views) if i % 8 != 0]
            test = [v for i, v in enumerate(views) if i % 8 == 0]
        else:
            train, test = views, []
    extent = nerfpp_radius(train)
    rng = random.Random(seed)
    if shuffle:
        rng.shuffle(train)
        rng.shuffle(test)

    def cams(lst):
        out = []
        for uid, v in enumerate(lst):
            # loadCam sizes from the image itself; COLMAP FoVs come from the camera's size in cameras.bin / .txt
            w, h = camera_resolution(*image_size(v.path), resolution)
            out.append(make_camera(v.R, v.T, v.FovX, v.FovY, w, h, uid))
        return out

    pcd, mesh, multi, clouds, flame = None, None, None, None, None
    if gs_type == "gs_multi_mesh":
        multi, clouds = multi_mesh_gaussians(source_path, list(meshes or []), list(num_splats), seed)
    elif gs_type == "gs_flame":
        flame = flame_init(flame_model, seed)
    elif kind == "blender":
        if gs_type == "gs_mesh":
            mesh = mesh_gaussians_from_obj(os.path.join(source_path, "mesh.obj"), num_splats, seed)
        elif os.path.exists(os.path.join(source_path, "points3d.ply")):
            pcd = io_ply.load_point_cloud(os.path.join(source_path, "points3d.ply"))
        else:
            pcd = scenes.random_point_cloud(100_000, seed)
    else:
        sparse = os.path.join(source_path, "sparse/0")
        if os.path.exists(os.path.join(sparse, "points3D.ply")):
            pcd = io_ply.load_point_cloud(os.path.join(sparse, "points3D.ply"))
        else:
            pcd = io_ply.point_cloud_arrays(io_ply.point_cloud_elements(*read_colmap_points(sparse)))
    return Scene(cams(train), cams(test), train, test, extent, pcd, mesh, multi, clouds, flame,
                 mode="RGBA" if kind == "blender" else "RGB", white_background=bool(white_background), _rng_state=rng.getstate())


def load_scene(source_path: str, gs_type: str, white_background: bool = False, eval: bool = False, resolution: int = -1,
               images: str = "images", num_splats=2, seed: int = 0, shuffle: bool = True, device="cuda",
               workers: Optional[int] = None, meshes: Optional[List[str]] = None, flame_model: str = DEFAULT_FLAME_MODEL) -> Scene:
    """A COLMAP (`sparse/` present) or NeRF-synthetic (`transforms_train.json`) scene as the reference's Scene(args) builds
    it for `gs_type`, with every ground-truth image prepared on `device` (uint8 [H,W,3], resident) and the cameras moved
    there.  `seed` plays safe_state's role: it seeds the shuffle / view-order stream, the random point cloud and the gs_mesh
    initialisation.  Images are decoded on `workers` host threads (default: up to 8); the result does not depend on it.
    meshes / flame_model: as read_scene."""
    sc = read_scene(source_path, gs_type, white_background, eval, resolution, images, num_splats, seed, shuffle, meshes, flame_model)
    if workers is None:
        workers = min(8, os.cpu_count() or 1)
    prep = GroundTruthPreparer(device)
    views = sc.train_views + sc.test_views
    cams = sc.train_cameras + sc.test_cameras
    out = []
    for v, cam, arr in zip(views, cams, _decoded([v.path for v in views], sc.mode, workers)):
        img = prep.upload(arr)
        if sc.mode == "RGBA":
            img = prep.composite(img, sc.white_background)
        out.append(prep.resize(img, cam.image_width, cam.image_height))
    n = len(sc.train_views)
    sc.train_images, sc.test_images = out[:n], out[n:]
    sc.train_cameras = [c.to(device) for c in sc.train_cameras]
    sc.test_cameras = [c.to(device) for c in sc.test_cameras]
    return sc
