"""The remote viewer's frames on the GPU: gms_image_clamp_u8 against ATen's `(torch.clamp(img, 0, 1) * 255).byte()
.permute(1, 2, 0)` byte for byte (random images, odd and one-pixel sizes, every k/255 and its neighbours, +-inf, NaN);
gms_b200.cli.view serving each of the six model types to a client thread over a socketpair, at two image sizes, two
scaling modifiers and both backgrounds, every image equal to the same camera rendered by a fresh renderer and converted
by ATen; a forced overflow that returns the same bytes; and exactly one host synchronisation per frame after a size's
first, counted under torch.cuda.set_sync_debug_mode("warn")."""
import argparse
import os
import socket
import threading
import warnings

import numpy as np
import pytest
import torch

import flame_driver
from gms_b200 import io_image, io_ply, network_gui, scenes
from gms_b200.cli import view
from gms_b200.flame import NativeFlame
from gms_b200.model import FlameGaussianModel, FreeGaussianModel, MeshGaussianModel, MultiMeshGaussianModel

pytestmark = pytest.mark.gpu
SOURCE = "/data/scenes/viewer"


def _aten(img):
    return (torch.clamp(img, 0, 1) * 255).byte().permute(1, 2, 0).contiguous()


def _edge_values() -> np.ndarray:
    k = (np.arange(256, dtype=np.float32) / np.float32(255)).astype(np.float32)
    half = ((np.arange(256, dtype=np.float64) + 0.5) / 255).astype(np.float32)
    special = np.array([-np.inf, np.inf, np.nan, -0.0, 0.0, 1.0, -1.0, 2.0, 1e30, -1e30, 1e-45, -1e-45, 1e-7, 0.5,
                        np.float32(1) - np.float32(2 ** -24), 1 + 2 ** -23], np.float32)
    nan_bits = np.array([0xFFC00000, 0x7F800001, 0xFFFFFFFF, 0x7FFFFFFF], np.uint32).view(np.float32)    # -NaN, payloads
    return np.concatenate([k, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(2)), half,
                           np.nextafter(half, np.float32(-1)), np.nextafter(half, np.float32(2)), special, nan_bits])


@pytest.mark.parametrize("shape", [(3, 1, 1), (3, 7, 333), (3, 64, 257), (1, 5, 9), (4, 3, 2), (3, 1080, 1920)])
def test_clamp_u8_equals_aten_on_random_images(shape):
    g = torch.Generator(device="cuda").manual_seed(sum(shape))
    for img in (torch.randn(shape, device="cuda", generator=g) * 0.7 + 0.5,
                torch.rand(shape, device="cuda", generator=g) * 2 - 0.5):
        got = io_image.clamp_u8(img)
        assert got.shape == (shape[1], shape[2], shape[0])
        assert torch.equal(got, _aten(img)), shape


@pytest.mark.parametrize("width", [1, 7, 255, 257])
def test_clamp_u8_equals_aten_at_the_edges(width):
    v = _edge_values()
    n = -(-v.size // (3 * width)) * 3 * width
    v = np.concatenate([v, np.resize(v, n - v.size)])
    img = torch.from_numpy(v).cuda().reshape(3, -1, width)
    got = io_image.clamp_u8(img)
    want = _aten(img)
    bad = (got != want).nonzero()
    assert bad.numel() == 0, [(img[c, y, x].item(), got[y, x, c].item(), want[y, x, c].item()) for y, x, c in bad[:8].tolist()]
    torch.cuda.synchronize()
    assert torch.isnan(img).any() and torch.isinf(img).any()


def _cfg(out, gs_type):
    os.makedirs(os.path.join(out, "point_cloud", "iteration_7"), exist_ok=True)
    cfg = argparse.Namespace(sh_degree=3, source_path=SOURCE, model_path=out, images="images", resolution=-1,
                             white_background=False, data_device="cuda", eval=True, num_splats=[2], meshes=[], gs_type=gs_type)
    with open(os.path.join(out, "cfg_args"), "w") as f:
        f.write(str(cfg))
    return os.path.join(out, "point_cloud", "iteration_7", "point_cloud.ply")


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    """gs_type -> model directory; gs_points reads the gs_flat checkpoint as a pseudo-mesh, as cli.render does."""
    d = tmp_path_factory.mktemp("viewer")
    out = {t: str(d / t) for t in ("gs_mesh", "gs_flat", "gs", "gs_multi_mesh", "gs_flame")}
    iv, ifc = scenes.icosphere(2, 0.8)
    io_ply.save_mesh_model(_cfg(out["gs_mesh"], "gs_mesh"), MeshGaussianModel.from_params(
        scenes.init_mesh_gaussians(iv, ifc, K=2, seed=0), "cuda", packed_features=True))
    g = scenes.flat_gaussians(2000, seed=4)
    FreeGaussianModel(g["means3D"] * 0.6, torch.log(g["scales"][:, 1:]).contiguous(), g["rotations"], g["shs"],
                      torch.logit(g["opacities"]), "gs_flat", "cuda", 3).save(_cfg(out["gs_flat"], "gs_flat"))
    s3 = g["scales"].clone()
    s3[:, 0] = s3[:, 1]
    FreeGaussianModel(g["means3D"] * 0.6, torch.log(s3), g["rotations"], g["shs"], torch.logit(g["opacities"]), "gs",
                      "cuda", 3).save(_cfg(out["gs"], "gs"))
    pa = scenes.init_mesh_gaussians(*scenes.icosphere(1, 0.5), K=2, seed=1)
    pb = scenes.init_mesh_gaussians(*scenes.torus(8, 6, R=0.7, r=0.15), K=3, seed=2)
    io_ply.save_multi_mesh_model(_cfg(out["gs_multi_mesh"], "gs_multi_mesh"),
                                 MultiMeshGaussianModel.from_mesh_params([pa, pb], "cuda", packed_features=True))
    torch.manual_seed(0)
    syn = flame_driver.SyntheticFlame(rings=23, segments=24).cuda()
    fl = NativeFlame(v_template=syn.v_template, shapedirs=syn.shapedirs, posedirs=syn.posedirs, J_regressor=syn.J_regressor,
                     parents=flame_driver.PARENTS, lbs_weights=syn.lbs_weights, faces=syn.faces)
    fm = FlameGaussianModel.create(fl, torch.from_numpy(np.asarray(syn.faces, np.int64)).cuda(), K=3, seed=3)
    io_ply.save_flame_model(_cfg(out["gs_flame"], "gs_flame"), fm, point_cloud=fl.to_point_cloud())
    out["gs_points"] = out["gs_flat"]
    return out


def _message(W, H, s, eye=(2.4, 0.8, 1.0)):
    """The request a viewer sends for a look_at camera: the matrices before network_gui's column negations."""
    cam = scenes.look_at_camera(eye, (0, 0, 0), W, H)
    wv, fp = cam.world_view_transform.clone(), cam.full_proj_transform.clone()
    wv[:, 1:3] = -wv[:, 1:3]
    fp[:, 1] = -fp[:, 1]
    return {"resolution_x": W, "resolution_y": H, "train": False, "fov_y": cam.FoVy, "fov_x": cam.FoVx, "z_near": 0.01,
            "z_far": 100.0, "shs_python": False, "rot_scale_python": False, "keep_alive": True, "scaling_modifier": s,
            "view_matrix": wv.reshape(-1).tolist(), "view_projection_matrix": fp.reshape(-1).tolist()}


def _expected(frames, msg) -> bytes:
    """The frame by a fresh renderer and ATen's conversion, train.py:72-74."""
    cam = network_gui.parse(msg).camera
    cam = cam.on(cam.packed().cuda())
    r = frames.renderer_cls(frames.model, cam.image_width, cam.image_height)
    return _aten(r.render(cam, frames.bg, scale_modifier=msg["scaling_modifier"])[0]).cpu().numpy().tobytes()


def _session(frames, verify, messages, draw=None):
    """Serves `messages` from a client thread over a socketpair; returns the replies (image bytes or None, verify)."""
    a, b = socket.socketpair()
    replies = []

    def client():
        try:
            for m in messages:
                replies.append(network_gui.request(a, m))
        finally:
            a.close()

    t = threading.Thread(target=client)
    t.start()
    network_gui.serve(b, draw or frames, verify, log=lambda s: None)
    t.join()
    return replies


def _counted(frames, syncs):
    """frames, with the host synchronisations of every frame but a size's first listed into `syncs` (where each was
    asked for)."""
    def draw(cam, s):
        if (cam.image_width, cam.image_height) not in frames.sizes:
            return frames(cam, s)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                out = frames(cam, s)
            finally:
                torch.cuda.set_sync_debug_mode(0)
        syncs.append([f"{x.filename}:{x.lineno}: {x.message}" for x in w if "called a synchronizing CUDA operation" in str(x.message)])
        return out
    return draw


@pytest.mark.parametrize("gs_type", ["gs_mesh", "gs_flat", "gs", "gs_points", "gs_multi_mesh", "gs_flame"])
def test_served_frames_equal_the_reference_conversion(models, gs_type):
    for white in (False, True):
        args, frames, verify = view.load(["-m", models[gs_type], "--gs_type", gs_type] + (["-w"] if white else []))
        assert verify == SOURCE.encode() and frames.bg.tolist() == [float(white)] * 3
        msgs = [_message(64, 48, 1.0), _message(37, 23, 1.0), {"resolution_x": 0, "resolution_y": 0},
                _message(64, 48, 0.6, eye=(0.5, 2.6, 0.9)), _message(37, 23, 0.6), _message(64, 48, 1.0, eye=(-2.0, 1.5, 1.2)),
                _message(37, 23, 1.0, eye=(0.3, -2.2, -1.4))]
        syncs = []
        with torch.no_grad():
            replies = _session(frames, verify, msgs, _counted(frames, syncs))
        assert len(replies) == len(msgs)
        for m, (image, v) in zip(msgs, replies):
            assert v == verify
            if m["resolution_x"] == 0:
                assert image is None
                continue
            want = _expected(frames, m)
            assert image == want, (gs_type, white, m["resolution_x"], m["scaling_modifier"])
            assert len(set(want[::3])) > 8, "the camera should see the model"
        assert [len(x) for x in syncs] == [1] * 4, syncs
        assert sum(r.overflows for r, _, _ in frames.sizes.values()) == 0


@pytest.mark.parametrize("gs_type", ["gs_mesh", "gs_points"])
def test_overflowed_frame_is_drawn_again(models, gs_type):
    _, frames, verify = view.load(["-m", models[gs_type], "--gs_type", gs_type])
    first, second = _message(64, 48, 1.0), _message(64, 48, 0.8, eye=(0.5, 2.6, 0.9))

    def force(cam, s):
        if (64, 48) in frames.sizes:
            frames.sizes[(64, 48)][0].capacity_override = 1
        return frames(cam, s)

    with torch.no_grad():
        replies = _session(frames, verify, [first, second], force)
    r = frames.sizes[(64, 48)][0]
    assert r.overflows == 1
    for m, (image, _) in zip([first, second], replies):
        assert image == _expected(frames, m)
