"""-m gpu: the sync-free training frame against the oracle.

NativeFrame(sync_free=True) runs every frame after the first through gms_train_frame with a PREDICTED binning capacity:
N stays on the device, the binning region is larger than N and its tail holds sentinel keys.  That is the path every
training step takes, and the synchronising rasterizer entry points (test_gpu_parity.py, where the capacity is N) never
reach it.  Here the second frame of a camera -- the first sync-free one -- is compared with the oracle chain (oracle
expansion -> oracle rasterizer, float64 loss gradient) under every binning, sort and compositing option, at image sizes on
both sides of the hand-written sort's pass boundary (T = 255 tiles: one 8-bit pass; T = 256: two) and at a ragged size.
An overflowed frame (N above the capacity) must render the background with zero gradients and be counted, and the next
frame of the same camera must be right again."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

import aten_reference
from gms_b200 import _lib, scenes
from gms_b200.model import MeshGaussianModel
from gms_b200.optim import FlatAdam, mesh_model_groups
from gms_b200.trainer import NativeFrame
from gpu_helpers import GRAD_TOL, assert_image_parity, oracle_chain
from helpers import settings_from_camera

pytestmark = pytest.mark.gpu

LAMBDA = 0.2
BG = (0.2, 0.5, 0.9)
SIZES = [(240, 272), (256, 256), (400, 300)]      # T = 15 x 17 = 255, 16 x 16 = 256, 25 x 19 = 475 (300 = 18.75 tiles)
OPTION_SETS = [{}, {"sort_impl": 1}, {"bin_impl": 1}, {"bin_impl": 1, "sort_impl": 1}, {"key16": 0}, {"key16": 0, "sort_impl": 1},
               {"composite_fwd": 3}, {"composite_bwd": 3}, {"tile_order": 0}, {"sh_staged": 0}, {"sh_staged": 2}]
GRADS = ("vertices", "_alpha", "_scale", "_opacity", "_features")

_scenes, _oracle = {}, {}


def _opt_id(opts):
    return ",".join(f"{k}={v}" for k, v in opts.items()) or "defaults"


def _scene(W, H):
    if (W, H) not in _scenes:
        p = scenes.init_mesh_gaussians(*scenes.icosphere(4), K=3, seed=21, trained_like=True)
        cam = scenes.look_at_camera((2.2, 0.7, 1.0), (0, 0, 0), W, H)
        gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(W * H))       # the ground truth: any fixed image
        _scenes[(W, H)] = (p, cam, gt)
    return _scenes[(W, H)]


class _Options:
    def __init__(self, opts):
        self.opts = opts

    def __enter__(self):
        self.old = {k: _lib.set_option(k, v) for k, v in self.opts.items()}

    def __exit__(self, *exc):
        for k, v in self.old.items():
            _lib.set_option(k, v)


def _new_frame(p, W, H):
    model = MeshGaussianModel.from_params(p, "cuda", packed_features=True)
    opt = FlatAdam(mesh_model_groups(model))            # owns the preallocated .grad buffers the frame writes
    return model, opt, NativeFrame(model, W, H, LAMBDA, sync_free=True)


def _frame_outputs(fr, P):
    """The frame's expansion outputs, radii and image, read from its workspace through gms_frame_views."""
    v = _lib.FrameView()
    _lib.check(_lib.lib().gms_frame_views(fr.ws.data_ptr(), P, fr.W, fr.H, C.byref(v)), "gms_frame_views")

    def take(ptr, shape, dtype=torch.float32):
        off = ptr - fr.ws.data_ptr()
        return fr.ws[off:off + 4 * int(np.prod(shape))].view(dtype).view(shape).cpu()

    return dict(xyz=take(v.xyz, (P, 3)), scales=take(v.scales, (P, 3)), rotations=take(v.rotations, (P, 4)),
                radii=take(v.radii, (P,), torch.int32), image=take(v.image, (3, fr.H, fr.W)),
                invdepth=take(v.invdepth, (1, fr.H, fr.W)))


def _run(fr, opt, cam, gt, bg):
    opt.zero_grad()
    loss = fr.run(cam, gt, bg).item()
    torch.cuda.synchronize()
    return loss


def _oracle_for(W, H, out, dC):
    """Oracle chain of one scene; reused for every option set that hands it the same Gaussians and the same dL/dimage
    (the options change how the kernels compute, not what)."""
    p, cam, _ = _scene(W, H)
    key = (W, H, hashlib.sha1(b"".join(out[k].numpy().tobytes() for k in ("xyz", "scales", "rotations")) + dC.tobytes()).hexdigest())
    if key not in _oracle:
        S = settings_from_camera(cam, bg=BG)
        _oracle[key] = oracle_chain(p, S, dC, (out["xyz"], out["scales"], out["rotations"]))
    return _oracle[key]


def _check_frame_against_oracle(model, fr, loss, gt, tag):
    W, H = fr.W, fr.H
    P = model._scale.shape[0]
    out = _frame_outputs(fr, P)
    # dL/dimage of the training loss in float64 at the frame's own image: the upstream gradient of the oracle backward
    img = out["image"].double().requires_grad_(True)
    aten_reference.training_loss(img, gt.double(), LAMBDA).backward()
    st, og = _oracle_for(W, H, out, img.grad.float().numpy())
    N = fr.last_num_rendered
    print(f"[native frame {tag}] {W}x{H} P={P} N={N} capacity={fr.capacity}")
    np.testing.assert_array_equal(out["radii"].numpy(), st.radii)
    assert N == st.N
    assert_image_parity(st, out["image"].numpy())
    with torch.no_grad():
        ref_loss = float(aten_reference.training_loss(torch.tensor(st.color, dtype=torch.float64), gt.double(), LAMBDA))
    print(f"[native frame {tag}] loss {loss:.8f}, float64 loss of the oracle image {ref_loss:.8f}, |diff| = {abs(loss - ref_loss):.2e}")
    assert abs(loss - ref_loss) <= 1e-5 * max(1.0, abs(ref_loss))
    fg = model._features.grad.detach().cpu()
    got = dict(vertices=model.vertices.grad, _alpha=model._alpha.grad, _scale=model._scale.grad, _opacity=model._opacity.grad,
               _features_dc=fg[:, :1], _features_rest=fg[:, 1:])
    msg = []
    for k, ref_g in og.items():
        scale = max(float(ref_g.abs().max()), 1e-20)
        e = float((got[k].detach().cpu().reshape(ref_g.shape).double() - ref_g.double()).abs().max()) / scale
        msg.append(f"{k} {e:.2e}")
        assert e <= GRAD_TOL.get(k, 2e-4), (k, e)
    print(f"[native frame {tag}] grad max err / max|ref|: " + ", ".join(msg))


@pytest.mark.parametrize("opts", OPTION_SETS, ids=_opt_id)
@pytest.mark.parametrize("W,H", SIZES)
def test_sync_free_frame_matches_oracle(W, H, opts):
    """The second frame of a camera (capacity predicted from the first, N on the device) against the oracle: radii and N
    bit-exact, image within 1e-5 outside the threshold-ambiguous pixels, loss and every parameter gradient."""
    p, cam, gt = _scene(W, H)
    cam_d, gt_d, bg = cam.to("cuda"), gt.cuda(), torch.tensor(BG, device="cuda")
    with _Options(opts):
        model, opt, fr = _new_frame(p, W, H)
        _run(fr, opt, cam_d, gt_d, bg)                          # synchronising: learns N
        n_first = fr.last_num_rendered
        loss = _run(fr, opt, cam_d, gt_d, bg)                   # sync-free: binning region sized by the prediction
    assert fr.overflows == 0 and fr.capacity > n_first > 0
    _check_frame_against_oracle(model, fr, loss, gt, _opt_id(opts))


@pytest.mark.parametrize("opts", [{}, {"sort_impl": 1}, {"key16": 0}, {"bin_impl": 1}, {"bin_impl": 1, "sort_impl": 1}], ids=_opt_id)
def test_overflowed_frame_renders_background_then_recovers(opts):
    """Capacity N - 1: the frame raises the overflow flag, renders the background, leaves every gradient zero and is
    counted in `overflows`; the camera's next frame, sized from the true N, matches the oracle."""
    W, H = SIZES[2]
    p, cam, gt = _scene(W, H)
    cam_d, gt_d, bg = cam.to("cuda"), gt.cuda(), torch.tensor(BG, device="cuda")
    with _Options(opts):
        model, opt, fr = _new_frame(p, W, H)
        _run(fr, opt, cam_d, gt_d, bg)
        N = fr.last_num_rendered
        fr.capacity_override = N - 1
        _run(fr, opt, cam_d, gt_d, bg)
        assert fr.last_num_rendered == N and fr.capacity == N - 1 and fr.overflows == 1
        out = _frame_outputs(fr, model._scale.shape[0])
        assert torch.equal(out["image"], torch.tensor(BG)[:, None, None].expand(3, H, W))
        assert float(out["invdepth"].abs().max()) == 0.0
        for k in GRADS:
            assert float(getattr(model, k).grad.abs().max()) == 0.0, k
        fr.capacity_override = None
        loss = _run(fr, opt, cam_d, gt_d, bg)
    assert fr.overflows == 1 and fr.capacity > N
    _check_frame_against_oracle(model, fr, loss, gt, "after overflow, " + _opt_id(opts))
