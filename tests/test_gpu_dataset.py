"""-m gpu: the dataset loader's device half.  gms_image_composite_rgba over every (value, alpha) pair and
gms_image_resize_u8 over down- and upscales against tests/resize_oracle.py, bit for bit, with canaries behind every output
and scratch buffer; load_scene against the reference's fixture (tests/golden/dataset.npz); trainers fed uint8 ground
truth against the same steps fed its dequantized float; and short training runs from load_scene."""
import ctypes as C
import hashlib
import json
import math
import os

import numpy as np
import pytest
import torch

import dataset_cases
import resize_oracle
from gms_b200 import _lib, dataset, io_image, scenes
from gms_b200.model import FreeGaussianModel, MeshGaussianModel
from gms_b200.render import NativeFreeRenderer
from gms_b200.trainer import FreeOptimizationParams, FreeTrainer, MeshTrainer
from helpers import random_gaussians

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "dataset.npz"))
CANARY = 0xA5
PAD = 4096


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _padded(n):
    """A device byte buffer of n + PAD bytes filled with the canary; -> (buffer, view of the first n)."""
    b = torch.full((n + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    return b, b[:n]


def _assert_canary(buf, n, what):
    tail = buf[n:].cpu()
    assert bool((tail == CANARY).all()), f"{what}: wrote past its end"


def test_composite_every_value_alpha_pair():
    v, a = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    rgba = np.stack([v, (v * 7) % 256, 255 - v, a], -1).astype(np.uint8)       # [256,256,4]
    src = torch.from_numpy(rgba).cuda()
    for white in (0, 1):
        buf, out = _padded(256 * 256 * 3)
        _lib.check(_lib.lib().gms_image_composite_rgba(src.data_ptr(), out.data_ptr(), 256, 256, white, _stream()), "composite")
        torch.cuda.synchronize()
        want = resize_oracle.composite(rgba, bool(white))
        assert np.array_equal(out.cpu().numpy().reshape(256, 256, 3), want), white
        _assert_canary(buf, out.numel(), "composite")


def test_composite_argument_checks():
    src = torch.zeros(16, dtype=torch.uint8, device="cuda")
    L = _lib.lib()
    assert L.gms_image_composite_rgba(src.data_ptr(), src.data_ptr(), 0, 2, 0, _stream()) == _lib.GMS_E_ARG
    assert L.gms_image_composite_rgba(src.data_ptr(), src.data_ptr(), 1, 2, 2, _stream()) == _lib.GMS_E_ARG
    assert L.gms_image_composite_rgba(src.data_ptr() + 1, src.data_ptr(), 1, 2, 0, _stream()) == _lib.GMS_E_ARG


def _resize_native(img: np.ndarray, w: int, h: int) -> np.ndarray:
    """gms_image_resize_u8 called directly, with canaries behind the output and the scratch."""
    H, W, _ = img.shape
    src = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    a = _lib.ResizeArgs()
    a.in_w, a.in_h, a.out_w, a.out_h, a.C = W, H, w, h, 3
    obuf, out = _padded(w * h * 3)
    a.src, a.dst = src.data_ptr(), out.data_ptr()
    keep = []
    sbuf, nscratch = None, 0
    if w != W:
        b, k = dataset.resize_coeffs(W, w)
        bt, kt = torch.from_numpy(b).cuda(), torch.from_numpy(k).cuda()
        keep += [bt, kt]
        a.bounds_h, a.coeffs_h, a.ksize_h = bt.data_ptr(), kt.data_ptr(), k.shape[1]
    if h != H:
        b, k = dataset.resize_coeffs(H, h)
        bt, kt = torch.from_numpy(b).cuda(), torch.from_numpy(k).cuda()
        keep += [bt, kt]
        a.bounds_v, a.coeffs_v, a.ksize_v = bt.data_ptr(), kt.data_ptr(), k.shape[1]
        a.row0, a.rows = int(b[0, 0]), int(b[-1, 0] + b[-1, 1] - b[0, 0])
        if w != W:
            nscratch = w * a.rows * 3
            sbuf, scr = _padded(nscratch)
            a.scratch, a.scratch_bytes = scr.data_ptr(), nscratch
    _lib.check(_lib.lib().gms_image_resize_u8(C.byref(a), _stream()), "gms_image_resize_u8")
    torch.cuda.synchronize()
    _assert_canary(obuf, w * h * 3, "resize output")
    if sbuf is not None:
        _assert_canary(sbuf, nscratch, "resize scratch")
    return out.cpu().numpy().reshape(h, w, 3)


RESIZE_CASES = [((800, 800), (400, 400)), ((512, 384), (128, 96)), ((512, 384), (64, 48)), ((4946, 3286), (1600, 1063)),
                ((1601, 37), (1599, 36)), ((37, 23), (18, 11)), ((333, 211), (160, 101)), ((64, 48), (80, 60)),
                ((101, 67), (101, 33)), ((101, 67), (50, 67)), ((30, 20), (31, 20)), ((90, 7), (1, 3)), ((40, 90), (13, 1)),
                ((9000, 9), (1600, 5)), ((7, 5), (7, 5))]


@pytest.mark.parametrize("src,dst", RESIZE_CASES, ids=[f"{s[0]}x{s[1]}-{d[0]}x{d[1]}" for s, d in RESIZE_CASES])
def test_resize_matches_oracle(src, dst):
    (W, H), (w, h) = src, dst
    img = np.random.default_rng(W * 7 + H).integers(0, 256, (H, W, 3), dtype=np.uint8)
    assert np.array_equal(_resize_native(img, w, h), resize_oracle.resize(img, w, h))


def test_resize_argument_checks():
    a = _lib.ResizeArgs()
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    a.in_w, a.in_h, a.out_w, a.out_h, a.C, a.src, a.dst = 4, 4, 2, 2, 3, buf.data_ptr(), buf.data_ptr()
    L = _lib.lib()
    assert L.gms_image_resize_u8(C.byref(a), _stream()) == _lib.GMS_E_ARG       # no tables
    a.C = 4
    assert L.gms_image_resize_u8(C.byref(a), _stream()) == _lib.GMS_E_ARG
    a.C, a.out_w = 3, 0
    assert L.gms_image_resize_u8(C.byref(a), _stream()) == _lib.GMS_E_ARG


@pytest.fixture(scope="module")
def datasets(tmp_path_factory):
    return dataset_cases.write_all(str(tmp_path_factory.mktemp("datasets")))


def _tree_digest(root):
    h = hashlib.sha256()
    for d, _, files in sorted(os.walk(root)):
        for f in sorted(files):
            p = os.path.join(d, f)
            h.update(os.path.relpath(p, root).encode() + open(p, "rb").read())
    return h.hexdigest()


@pytest.mark.parametrize("case", sorted(dataset_cases.CASES))
@pytest.mark.parametrize("workers", [1, 4])
def test_load_scene_matches_reference(case, workers, datasets):
    ds, kw = dataset_cases.CASES[case]
    before = _tree_digest(datasets[ds])
    sc = dataset.load_scene(datasets[ds], workers=workers, **kw)
    torch.cuda.synchronize()
    assert _tree_digest(datasets[ds]) == before
    g = {k[len(case) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(case + "/")}
    assert sc.view_order(40) == g["order"].tolist()
    for split, cams, imgs in (("train", sc.train_cameras, sc.train_images), ("test", sc.test_cameras, sc.test_images)):
        assert sc.train_names == g["train/names"].tolist() and sc.test_names == g["test/names"].tolist()
        assert len(imgs) == len(cams) == len(g[f"{split}/names"])
        for i, (c, img) in enumerate(zip(cams, imgs)):
            assert img.is_cuda and img.dtype == torch.uint8
            assert np.array_equal(img.cpu().numpy(), g[f"{split}/image{i}"]), (split, i)
            assert c.world_view_transform.is_cuda and (c.image_width, c.image_height) == tuple(g[f"{split}/size"][i])


def _mesh_model(seed=3):
    p = scenes.init_mesh_gaussians(*scenes.icosphere(2, 0.9), K=3, seed=seed)
    return MeshGaussianModel.from_params(p, "cuda", packed_features=True)


def _u8_views(n, W, H, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8).cuda() for _ in range(n)]


def _assert_within_run_to_run(a, b, c, what):
    """a (uint8 arm) against b (float arm) no further apart than 10x the distance of two float arms b, c: the frames
    accumulate vertex gradients and loss partial sums with float atomics, so two float runs differ in the last bits."""
    ab, bc = float((a - b).abs().max()), float((b - c).abs().max())
    assert ab <= 10 * bc + 1e-7, f"{what}: |uint8 - float| {ab:.3e} against float run-to-run {bc:.3e}"


def _check_gt_buffer(frame, fl):
    """the frame's dequantized ground truth is bit for bit the float ground truth of the other arm"""
    assert torch.equal(frame._gt_u8.buf, fl)


def test_mesh_trainer_uint8_equals_float():
    """50 native steps (and 5 of the autograd arm) fed uint8 ground truth against the same steps fed byte / 255: the frame
    sees the same float ground truth bit for bit, and losses and parameters stay within the float arm's run-to-run
    difference."""
    W, H = 96, 64
    cams = [c.to("cuda") for c in scenes.ring_cameras(4, 2.6, W, H)]
    for i, c in enumerate(cams):
        c.uid = i
    u8 = _u8_views(4, W, H)
    fl = [io_image.to_device_float(x).clone() for x in u8]
    bg = torch.zeros(3, device="cuda")
    for native, steps in ((True, 50), (False, 5)):
        models = [_mesh_model() for _ in range(3)]
        tr = [MeshTrainer(m, bg, native=native) for m in models]
        losses = [[], [], []]
        for it in range(steps):
            for k, t in enumerate(tr):
                losses[k].append(t.step(cams[it % 4], (u8 if k == 0 else fl)[it % 4]).clone())
            if native:
                _check_gt_buffer(tr[0]._frame, fl[it % 4])
            else:
                assert torch.equal(tr[0]._gt_u8.buf, fl[it % 4])
        _assert_within_run_to_run(*(torch.stack(l) for l in losses), f"losses native={native}")
        for n in ("vertices", "_alpha", "_scale", "_features", "_opacity"):
            _assert_within_run_to_run(*(getattr(m, n).detach() for m in models), f"{n} native={native}")


def test_free_trainer_uint8_equals_float():
    W, H = 96, 64
    cams = [c.to("cuda") for c in scenes.ring_cameras(4, 2.6, W, H)]
    for i, c in enumerate(cams):
        c.uid = i
    u8 = _u8_views(4, W, H, seed=1)
    fl = [io_image.to_device_float(x).clone() for x in u8]
    bg = torch.zeros(3, device="cuda")
    pts, colors, _ = scenes.random_point_cloud(3000, 0)
    models = [FreeGaussianModel.from_point_cloud(pts, colors, "gs_flat") for _ in range(3)]
    o = FreeOptimizationParams(iterations=50, densify_until_iter=0)
    tr = [FreeTrainer(m, bg, 2.0, o) for m in models]
    losses = [[], [], []]
    for it in range(50):
        for k, t in enumerate(tr):
            losses[k].append(t.step(cams[it % 4], (u8 if k == 0 else fl)[it % 4]).clone())
        _check_gt_buffer(tr[0].frame, fl[it % 4])
    _assert_within_run_to_run(*(torch.stack(l) for l in losses), "losses")
    for n in FreeGaussianModel.NAMES:
        _assert_within_run_to_run(*(getattr(m, n).detach() for m in models), n)


def _write_rendered_blender(root, W=128, n_train=12, n_test=4):
    """A NeRF-synthetic dataset of RGBA views (alpha 255) rendered by the native renderer from a known gs_flat model."""
    os.makedirs(os.path.join(root, "train"), exist_ok=True)
    os.makedirs(os.path.join(root, "test"), exist_ok=True)
    ring = scenes.ring_cameras(n_train + n_test, 3.0, W, W, elevation_deg=25.0)
    g = random_gaussians(2000, seed=21, extent=0.45, flat_frac=0.0)     # mostly background: the random cloud's fog must go
    target = FreeGaussianModel(g["means3D"], torch.log(g["scales"][:, 1:]).contiguous(), g["rotations"], g["shs"],
                               torch.logit(g["opacities"]), "gs_flat", "cuda", 0)
    r = NativeFreeRenderer(target, W, W)
    bg = torch.zeros(3, device="cuda")
    for split, cams in (("train", ring[:n_train]), ("test", ring[n_train:])):
        frames = []
        for i, c in enumerate(cams):
            img = r.render(c.to("cuda"), bg)[0]
            rgb = io_image.quantize(img).cpu().numpy().reshape(W, W, 3)
            dataset_cases.write_png(os.path.join(root, split, f"r_{i}.png"),
                                    np.concatenate([rgb, np.full((W, W, 1), 255, np.uint8)], 2))
            c2w = np.linalg.inv(c.world_view_transform.numpy().T.astype(np.float64))
            c2w[:3, 1:3] *= -1
            frames.append({"file_path": f"./{split}/r_{i}", "transform_matrix": c2w.tolist()})
        with open(os.path.join(root, f"transforms_{split}.json"), "w") as f:
            json.dump({"camera_angle_x": scenes.NERF_FOVX, "frames": frames}, f)
    v, fcs = scenes.icosphere(2, 0.7)
    with open(os.path.join(root, "mesh.obj"), "w") as f:
        for x in v:
            f.write("v %.6f %.6f %.6f\n" % tuple(x))
        for t in fcs + 1:
            f.write("f %d %d %d\n" % tuple(t))


def test_end_to_end_training_from_load_scene(tmp_path):
    """gs_flat from load_scene's random cloud for 300 iterations in view_order: the mean test PSNR rises by >= 3 dB; then a
    gs_mesh scene from the same files for 100 iterations: the loss stays finite and falls."""
    root = str(tmp_path / "scene")
    _write_rendered_blender(root)
    sc = dataset.load_scene(root, "gs_flat", eval=True)
    assert len(sc.train_cameras) == 12 and len(sc.test_cameras) == 4
    pts, colors, _ = sc.point_cloud
    model = FreeGaussianModel.from_point_cloud(pts, colors, "gs_flat")
    bg = torch.zeros(3, device="cuda")
    tr = FreeTrainer(model, bg, sc.cameras_extent, FreeOptimizationParams(iterations=300))
    psnr0 = float(tr.evaluate(sc.test_cameras, sc.test_images).mean[2])
    for v in sc.view_order(300):
        tr.step(sc.train_cameras[v], sc.train_images[v])
    psnr1 = float(tr.evaluate(sc.test_cameras, sc.test_images).mean[2])
    print(f"[load_scene gs_flat] test PSNR {psnr0:.2f} -> {psnr1:.2f} dB")
    assert psnr1 >= psnr0 + 3.0

    sm = dataset.load_scene(root, "gs_mesh", eval=True, num_splats=2)
    m = MeshGaussianModel.from_params(sm.mesh, "cuda", packed_features=True, active_sh_degree=0)
    mt = MeshTrainer(m, bg, native=True)
    losses = torch.stack([mt.step(sm.train_cameras[v], sm.train_images[v]).clone() for v in sm.view_order(100)]).cpu()
    assert bool(torch.isfinite(losses).all())
    first, last = float(losses[:10].mean()), float(losses[-10:].mean())
    print(f"[load_scene gs_mesh] loss {first:.4f} -> {last:.4f}")
    assert last < first
