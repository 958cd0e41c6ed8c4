"""-m gpu: the forward-only render frame (gms_render_frame through NativeRenderer) and the view metrics (gms_image_metrics,
NativeRenderer.evaluate).

1. The sync-free render of a camera equals, bit for bit, the forward outputs of the sync-free training frame for the same
   parameters and camera, under every binning / sort / compositing option that changes how the forward runs.
2. It matches the oracle at every active SH degree, with antialiasing and a scale modifier, and along an animated sweep.
3. An overflowed render gives the background and is counted; the camera's next render is right again.
4. A forward-only render requests no survivor-list space.
5. gms_image_metrics matches the reference's metrics (metrics.npz) and the float64 restatement, and is deterministic.
6. evaluate() matches a per-view loop of the autograd-shim render + the restatement; 8-bit ground truth gives the same
   bits as its float image; overflowed views are re-run and give the bits of a clean run."""
import math
import os

import numpy as np
import pytest
import torch

from gms_b200 import _lib, io_image, scenes
from gms_b200.metrics import image_metrics
from gms_b200.model import MeshGaussianModel
from gms_b200.render import NativeRenderer
from gms_b200.trainer import render_frame
from gpu_helpers import assert_image_parity
from helpers import settings_from_camera
from metrics_restated import metrics64
from oracle import expansion as oexp
from oracle import raster
from test_gpu_native_frame import SIZES, _frame_outputs, _new_frame, _Options, _run, _scene

pytestmark = pytest.mark.gpu

BG = (0.2, 0.5, 0.9)
FWD_OPTION_SETS = [{}, {"sort_impl": 1}, {"bin_impl": 1}, {"key16": 0}, {"composite_fwd": 3}, {"tile_order": 0}]
L1_SSIM_TOL, PSNR_TOL = 2e-6, 1e-4


def _opt_id(opts):
    return ",".join(f"{k}={v}" for k, v in opts.items()) or "defaults"


def _model(p, degree=3):
    return MeshGaussianModel.from_params(p, "cuda", packed_features=True, active_sh_degree=degree)


def _oracle(p, model, cam, degree=3, scale_modifier=1.0, antialiasing=False):
    """The oracle rasterizer on the model's own expansion of its current vertices (as oracle_chain: integer outputs compare
    bit for bit), with the oracle's opacities and SH features."""
    with torch.no_grad():
        xyz, sc, rot = (t.cpu() for t in model.expand_fused(activated=True))
    oxyz, sl, rr, _, _ = oexp.expand(model.vertices.detach().cpu(), p.faces, p._alpha, p._scale)
    osc, _, op, fe = oexp.activate(sl, rr, p._opacity, p._features_dc, p._features_rest)
    assert float((xyz - oxyz.detach()).abs().max()) <= 2e-6 and float(((sc - osc.detach()).abs() / osc.detach()).max()) <= 1e-5
    S = settings_from_camera(cam, sh_degree=degree, bg=BG, scale_modifier=scale_modifier, antialiasing=antialiasing)
    return raster.forward(S, xyz, op.detach(), shs=fe.detach().contiguous(), scales=sc, rotations=rot)


def _render_twice(r, cam, bg, **kw):
    r.render(cam, bg, **kw)                      # synchronising: learns N
    out = [t.clone() for t in r.render(cam, bg, **kw)]      # sync-free
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("opts", FWD_OPTION_SETS, ids=_opt_id)
@pytest.mark.parametrize("W,H", SIZES)
def test_render_is_bit_identical_to_the_training_frame_forward(W, H, opts):
    p, cam, gt = _scene(W, H)
    cam_d, gt_d, bg = cam.to("cuda"), gt.cuda(), torch.tensor(BG, device="cuda")
    with _Options(opts):
        model, opt, fr = _new_frame(p, W, H)
        _run(fr, opt, cam_d, gt_d, bg)
        _run(fr, opt, cam_d, gt_d, bg)              # sync-free training frame (no optimizer step: the parameters stay)
        ref = _frame_outputs(fr, model._scale.shape[0])
        r = NativeRenderer(model, W, H)
        image, radii, invd = _render_twice(r, cam_d, bg)
    assert r.overflows == 0 and r.capacity > 0
    assert r.last_num_rendered == fr.last_num_rendered
    assert torch.equal(image.cpu(), ref["image"])
    assert torch.equal(invd.cpu(), ref["invdepth"])
    assert torch.equal(radii.cpu(), ref["radii"])


@pytest.mark.parametrize("degree,scale_modifier,antialiasing", [(0, 1.0, False), (1, 1.0, False), (2, 1.0, False), (3, 1.0, False),
                                                                 (3, 1.3, False), (3, 1.0, True)])
def test_render_matches_the_oracle(degree, scale_modifier, antialiasing):
    W, H = SIZES[2]
    p, cam, _ = _scene(W, H)
    model = _model(p, degree)
    r = NativeRenderer(model, W, H)
    image, radii, _ = _render_twice(r, cam.to("cuda"), torch.tensor(BG, device="cuda"), scale_modifier=scale_modifier,
                                    antialiasing=antialiasing)
    st = _oracle(p, model, cam, degree, scale_modifier, antialiasing)
    np.testing.assert_array_equal(radii.cpu().numpy(), st.radii)
    assert r.last_num_rendered == st.N
    assert_image_parity(st, image.cpu().numpy())


def test_animated_sweep_matches_the_oracle():
    """scripts/render_time_animated.py:82-84: the caller moves the vertices, each frame re-expands from them."""
    W, H = SIZES[2]
    p, cam, _ = _scene(W, H)
    model = _model(p)
    r = NativeRenderer(model, W, H)
    cam_d, bg = cam.to("cuda"), torch.tensor(BG, device="cuda")
    v0 = model.vertices.detach().clone()
    r.render(cam_d, bg)
    for t in np.linspace(0.0, 10 * math.pi, 4):
        with torch.no_grad():
            model.vertices.data.copy_(scenes.transform_hotdog_fly(v0, float(t)))
        image, radii, _ = r.render(cam_d, bg)
        st = _oracle(p, model, cam)
        np.testing.assert_array_equal(radii.cpu().numpy(), st.radii)
        assert_image_parity(st, image.cpu().numpy())
    assert r.overflows == 0


@pytest.mark.parametrize("opts", [{}, {"bin_impl": 1}], ids=_opt_id)
def test_overflowed_render_gives_the_background_then_recovers(opts):
    W, H = SIZES[2]
    p, cam, _ = _scene(W, H)
    cam_d, bg = cam.to("cuda"), torch.tensor(BG, device="cuda")
    with _Options(opts):
        r = NativeRenderer(_model(p), W, H)
        good = _render_twice(r, cam_d, bg)
        N = r.last_num_rendered
        r.capacity_override = N - 1
        image, _, invd = r.render(cam_d, bg)
        torch.cuda.synchronize()
        assert r.last_num_rendered == N and r.capacity == N - 1 and r.overflows == 1
        assert torch.equal(image.cpu(), torch.tensor(BG)[:, None, None].expand(3, H, W))
        assert float(invd.abs().max()) == 0.0
        r.capacity_override = None
        again = [t.clone() for t in r.render(cam_d, bg)]
        torch.cuda.synchronize()
    assert r.overflows == 1 and r.capacity > N
    for a, b in zip(again, good):
        assert torch.equal(a, b)


@pytest.mark.parametrize("opts", [{}, {"bin_impl": 1}], ids=_opt_id)
def test_forward_only_render_requests_no_survivor_lists(opts):
    """At the same capacity the training frame's binning request holds the point list plus four survivor lists of 4 B per
    duplicate; the render's holds the point list only."""
    W, H = SIZES[2]
    p, cam, gt = _scene(W, H)
    cam_d, gt_d, bg = cam.to("cuda"), gt.cuda(), torch.tensor(BG, device="cuda")
    with _Options(opts):
        model, opt, fr = _new_frame(p, W, H)
        r = NativeRenderer(model, W, H)
        _render_twice(r, cam_d, bg)
        cap = r.capacity
        _run(fr, opt, cam_d, gt_d, bg)
        fr.capacity_override = cap
        _run(fr, opt, cam_d, gt_d, bg)
    req_render = r._scratch["requested"][_lib.BUF_BINNING]
    req_train = fr._scratch["requested"][_lib.BUF_BINNING]
    print(f"[render] capacity {cap}: binning request {req_render} B (render) vs {req_train} B (training frame)")
    assert req_train - req_render >= 16 * cap


def _check_metrics(got, ref, what):
    got = [float(v) for v in got]
    assert abs(got[0] - ref[0]) <= L1_SSIM_TOL and abs(got[1] - ref[1]) <= L1_SSIM_TOL, (what, got, ref)
    for k in (2, 3):
        if math.isinf(ref[k]):
            assert math.isinf(got[k]) and got[k] > 0, (what, k, got)
        else:
            assert abs(got[k] - ref[k]) <= PSNR_TOL, (what, k, got[k], ref[k])


@pytest.mark.parametrize("protocol", ["training_report", "metrics"])
def test_image_metrics_match_the_reference_fixture(golden_dir, protocol):
    d = np.load(os.path.join(golden_dir, "metrics.npz"))
    for i in range(int(d["n_cases"])):
        img, gt = torch.from_numpy(d[f"case{i}_img"]).cuda(), torch.from_numpy(d[f"case{i}_gt"]).cuda()
        _check_metrics(image_metrics(img, gt, protocol).cpu(), d[f"case{i}_{protocol}"], f"case{i}")


@pytest.mark.parametrize("protocol", ["training_report", "metrics"])
@pytest.mark.parametrize("H,W", [(1080, 1920), (201, 333), (32, 32), (7, 5)])
def test_image_metrics_match_the_restatement_and_are_deterministic(H, W, protocol):
    g = torch.Generator().manual_seed(H * W)
    img = torch.rand(3, H, W, generator=g) * 1.2 - 0.1
    gt = img + 0.1 * torch.randn(3, H, W, generator=g)
    a = image_metrics(img.cuda(), gt.cuda(), protocol).cpu()
    b = image_metrics(img.cuda(), gt.cuda(), protocol).cpu()
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))
    _check_metrics(a, metrics64(img, gt, protocol), f"{W}x{H}")
    same = image_metrics(img.cuda(), img.cuda(), protocol).cpu()
    assert same[2] == math.inf and same[3] == math.inf and same[0] == 0.0


def _views(n, W, H):
    p, _, _ = _scene(W, H)
    cams = [c.to("cuda") for c in scenes.ring_cameras(n, 2.6, W, H)]
    g = torch.Generator().manual_seed(5)
    gts8 = [(torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).cuda() for _ in range(n)]
    return p, cams, gts8


def test_evaluate_matches_the_reference_protocol():
    W, H = SIZES[2]
    p, cams, gts8 = _views(6, W, H)
    gts = [io_image.to_device_float(t).clone() for t in gts8]
    bg = torch.tensor(BG, device="cuda")
    model = _model(p)
    for protocol in ("training_report", "metrics"):
        res = NativeRenderer(model, W, H).evaluate(cams, gts, bg, protocol=protocol)
        assert res.per_view.shape == (6, 4)
        with torch.no_grad():
            for v, (cam, gt) in enumerate(zip(cams, gts)):
                image = render_frame(model, cam, bg)[0]
                _check_metrics(res.per_view[v], metrics64(image, gt, protocol), f"{protocol} view {v}")
        assert torch.equal(res.mean, res.per_view.mean(0))


def test_evaluate_u8_ground_truth_and_overflow_reruns_give_the_same_bits():
    W, H = SIZES[2]
    p, cams, gts8 = _views(6, W, H)
    gts = [io_image.to_device_float(t).clone() for t in gts8]
    bg = torch.tensor(BG, device="cuda")
    model = _model(p)
    clean = NativeRenderer(model, W, H).evaluate(cams, gts, bg)
    assert clean.rerun == []
    r8 = NativeRenderer(model, W, H)
    from_u8 = r8.evaluate(cams, gts8, bg)
    assert torch.equal(from_u8.per_view.view(torch.int64), clean.per_view.view(torch.int64))
    # a capacity between the smallest and the largest N of the set: some views overflow on the first pass
    ns = sorted(r8._view_n[r8._view_key(c)][0] for c in cams)
    assert ns[0] < ns[-1]
    r = NativeRenderer(model, W, H)
    r.capacity_override = (ns[0] + ns[-1]) // 2
    res = r.evaluate(cams, gts8, bg)
    print(f"[evaluate] N per view {ns}, capacity {r.capacity_override}: re-ran views {res.rerun}")
    assert res.rerun and r.overflows == len(res.rerun)
    assert torch.equal(res.per_view.view(torch.int64), clean.per_view.view(torch.int64))
