"""CPU: training on scenes whose views differ in size.  A frame sized for its largest view runs a smaller view in the same
workspace, which is sound only while every workspace and scratch layout of the smaller size fits inside the larger
one's; the library's byte counts are checked for that over a grid of sizes.  Mixed-size NeRF-synthetic and two-camera
COLMAP scenes load with the reference readers' per-view sizes and FoVs, and cli.train prepares a run on them, sizing the
trainer for the largest training view."""
import ctypes as C
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import mixed_sizes_cases as cases
from gms_b200 import _lib, dataset, io_image
from gms_b200.cli import train as cli_train

SIDES = [1, 2, 15, 16, 17, 31, 33, 100, 240, 256, 272, 1079, 1080, 1081, 1920, 4096]
PS = [0, 1, 1000, 1_000_000]
BASE = 1 << 20      # stand-in workspace address (gms_frame_views only computes offsets)


def _scratch(P, W, H):
    g, i = C.c_size_t(0), C.c_size_t(0)
    assert _lib.lib().gms_scratch_bytes(P, W, H, C.byref(g), C.byref(i)) == _lib.GMS_OK
    return g.value, i.value


def _loss(W, H):
    b = C.c_size_t(0)
    assert _lib.lib().gms_loss_scratch_bytes(3, H, W, C.byref(b)) == _lib.GMS_OK
    return b.value


@pytest.mark.parametrize("P", PS)
def test_workspace_and_scratch_grow_with_width_and_height(P):
    """The training-frame workspace, the rasterizer's geometry and per-pixel scratch and the loss scratch never shrink when
    the width or the height grows: along each axis of the grid every byte count is at most its neighbour's."""
    L = _lib.lib()
    ws = np.array([[L.gms_frame_workspace_bytes(P, W, H) for H in SIDES] for W in SIDES], dtype=np.int64)
    sc = np.array([[_scratch(P, W, H) for H in SIDES] for W in SIDES], dtype=np.int64)
    loss = np.array([[_loss(W, H) for H in SIDES] for W in SIDES], dtype=np.int64)
    for name, a in (("frame workspace", ws), ("geometry scratch", sc[..., 0]), ("image scratch", sc[..., 1]), ("loss scratch", loss)):
        assert (np.diff(a, axis=0) >= 0).all() and (np.diff(a, axis=1) >= 0).all(), name
    assert (sc[..., 0] == sc[0, 0, 0]).all()        # the geometry scratch depends on P alone
    # binning scratch depends on N alone, which the capacity prediction sizes per view
    assert L.gms_binning_bytes(1 << 20, P) == L.gms_binning_bytes(1 << 20, P + 7)


@pytest.mark.parametrize("P", [1, 1000])
def test_every_frame_view_of_a_smaller_size_lies_inside_the_larger_workspace(P):
    """gms_frame_views at w x h <= W x H: the image [3,h,w] and the inverse depth [h,w] end inside the W x H workspace, and the
    size-independent rows (xyz, scales, rotations, opacities, radii) sit where the W x H frame has them."""
    L = _lib.lib()
    for W, H in [(1920, 1080), (1080, 1920), (256, 256), (33, 17)]:
        end = BASE + L.gms_frame_workspace_bytes(P, W, H)
        big = _lib.FrameView()
        assert L.gms_frame_views(BASE, P, W, H, C.byref(big)) == _lib.GMS_OK
        for w in [1, 16, W // 2, W]:
            for h in [1, 16, H // 2, H]:
                v = _lib.FrameView()
                assert L.gms_frame_views(BASE, P, w, h, C.byref(v)) == _lib.GMS_OK
                assert v.image + 12 * w * h <= end and v.invdepth + 4 * w * h <= end, (W, H, w, h)
                for n in ("xyz", "scales", "rotations", "opacities", "radii"):
                    assert getattr(v, n) == getattr(big, n), (n, W, H, w, h)


def test_ground_truth_buffer_takes_smaller_images_only_when_up_to():
    """The ground-truth buffer of an exact-size frame refuses any other size; an up_to one refuses only a larger image
    (both before any device work)."""
    exact = io_image.GroundTruthBuffer(32, 48, "cpu")
    up_to = io_image.GroundTruthBuffer(32, 48, "cpu", up_to=True)
    for shape in [(48, 32, 3), (16, 48, 3)]:
        with pytest.raises(ValueError, match=r"must be \[32,48,3\]"):
            exact(torch.zeros(shape, dtype=torch.uint8), "test")
    for shape in [(33, 48, 3), (32, 49, 3), (48, 32, 3), (32, 48, 4)]:
        with pytest.raises(ValueError, match=r"must be at most \[32,48,3\]"):
            up_to(torch.zeros(shape, dtype=torch.uint8), "test")


# ------------------------------------------------------------------------------------------------ scenes and the CLI

def _focal2fov(f, n):
    return 2 * math.atan(n / (2 * f))


@pytest.fixture(scope="module")
def roots(tmp_path_factory):
    base = tmp_path_factory.mktemp("mixed")
    return {"blender": cases.write_blender(str(base / "blender")), "colmap": cases.write_colmap(str(base / "colmap"))}


def test_blender_views_keep_their_own_size_and_fov(roots):
    """readCamerasFromTransforms: each view's size is its PNG's; FovY = focal2fov(fov2focal(FovX, width), height)."""
    sc = dataset.read_scene(roots["blender"], "gs_flat", eval=True, shuffle=False)
    want = [cases.LANDSCAPE, cases.PORTRAIT] * 3
    assert [(c.image_width, c.image_height) for c in sc.train_cameras] == want
    assert [(c.image_width, c.image_height) for c in sc.test_cameras] == want[:2]
    for v, c in zip(sc.train_views + sc.test_views, sc.train_cameras + sc.test_cameras):
        fovy = _focal2fov(v.width / (2 * math.tan(v.FovX / 2)), v.height)
        assert (v.width, v.height) == (c.image_width, c.image_height)
        assert v.FovY == pytest.approx(fovy, rel=1e-12) and c.FoVy == pytest.approx(fovy, rel=1e-12)


def test_colmap_views_take_their_cameras_size_and_fov(roots):
    """readColmapCameras: each image takes its camera's size, FovX = focal2fov(fx, width), FovY = focal2fov(fy, height)."""
    sc = dataset.read_scene(roots["colmap"], "gs_flat", eval=False, shuffle=False)
    cams = {cid: (size, p) for cid, _, size, p in cases.colmap_cameras()}
    assert len(sc.train_cameras) == 16
    for v, c in zip(sc.train_views, sc.train_cameras):
        k = int(v.name.split("_")[1])
        (W, H), p = cams[1 + cases.camera_of(k)]
        fx, fy = (p[0], p[1]) if cases.camera_of(k) == 0 else (p[0], p[0])
        assert (v.width, v.height) == (c.image_width, c.image_height) == (W, H), v.name
        assert c.FoVx == pytest.approx(_focal2fov(fx, W), rel=1e-12) and c.FoVy == pytest.approx(_focal2fov(fy, H), rel=1e-12)


class _Stub:
    """Stands in for a model or trainer class: records its keyword arguments (the models and trainers need a GPU)."""
    def __init__(self, *a, **k):
        self.kwargs = k
        self.opt = SimpleNamespace(groups=[])

    @classmethod
    def create(cls, *a, **k):
        return cls()

    from_params = from_mesh_params = from_point_cloud = create


@pytest.mark.parametrize("gs_type,kind", [("gs_mesh", "blender"), ("gs", "blender"), ("gs_flat", "colmap"),
                                          ("gs_multi_mesh", "colmap")])
def test_prepare_sizes_the_trainer_for_the_largest_training_view(roots, gs_type, kind, tmp_path, monkeypatch):
    """parse_args and prepare() accept a mixed-size scene and hand the trainer the largest training width and height."""
    for name in ("MeshGaussianModel", "MultiMeshGaussianModel", "FreeGaussianModel", "MeshTrainer", "FreeTrainer"):
        monkeypatch.setattr(cli_train, name, _Stub)
    monkeypatch.setattr(cli_train, "open_summary_writer", lambda path, log: None)
    extra = ["--meshes", *cases.MESHES, "--num_splats", *map(str, cases.NUM_SPLATS)] if gs_type == "gs_multi_mesh" else []
    args = cli_train.parse_args(["-s", roots[kind], "-m", str(tmp_path / "out"), "--gs_type", gs_type, "--eval", "--quiet"] + extra)
    sc = dataset.read_scene(roots[kind], gs_type, eval=True, meshes=args.meshes,
                            num_splats=args.num_splats if gs_type == "gs_multi_mesh" else args.num_splats[0])
    assert len({(c.image_width, c.image_height) for c in sc.train_cameras}) == 2
    run = cli_train.Training(args, device="cpu", scene=sc).prepare()
    W = max(c.image_width for c in sc.train_cameras)
    H = max(c.image_height for c in sc.train_cameras)
    assert (W, H) == (48, 48) and cli_train.training_size(sc) == (W, H)
    assert run.trainer.kwargs["max_size"] == (W, H)
