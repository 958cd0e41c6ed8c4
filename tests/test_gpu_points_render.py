"""-m gpu: the forward-only gs_points (pseudo-mesh) render frame, gms_points_render_frame through PointsRenderer.

1. The render matches the oracle chain (the pseudo-mesh expansion of oracle/expansion.py, sigmoid, the oracle rasterizer) at
   every active SH degree, with antialiasing, with a scale modifier, and on triangles moved by transform_hotdog.
2. It is bit-identical to the autograd-shim render of the same triangles (render_points_frame).
3. The sync-free render of a view is bit-identical to its synchronising render under every binning / sort / compositing
   option that changes how the forward runs.
4. An overflowed render gives the background and is counted; the view's next render is right again.
5. A forward-only render requests no survivor-list space.
6. A gs_flat checkpoint loads to the pseudo-mesh that points_prepare_vertices (and the reference) build from it.
7. evaluate() matches a per-view loop of render + image_metrics; 8-bit ground truth and overflow re-runs give the same bits.
8. A `triangles` override renders those triangles and leaves the model untouched.
9. Bad arguments are refused with GMS_E_ARG before anything is launched."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from gms_b200 import _lib, expansion, io_image, io_ply, scenes
from gms_b200.metrics import image_metrics
from gms_b200.model import MeshGaussianModel, PointsModel
from gms_b200.render import PointsRenderer, render_points_frame
from gpu_helpers import assert_image_parity
from helpers import settings_from_camera
from oracle import expansion as oexp
from oracle import raster

pytestmark = pytest.mark.gpu

BG = (0.2, 0.5, 0.9)
W, H = 400, 300
FWD_OPTION_SETS = [{}, {"sort_impl": 1}, {"bin_impl": 1}, {"key16": 0}, {"composite_fwd": 3}, {"tile_order": 0}]
HOTDOG_TIMES = (0.0, 1.7, 10 * math.pi * 43 / 99)

_params = {}


def _opt_id(opts):
    return ",".join(f"{k}={v}" for k, v in opts.items()) or "defaults"


class _Options:
    def __init__(self, opts):
        self.opts = opts

    def __enter__(self):
        self.old = {k: _lib.set_option(k, v) for k, v in self.opts.items()}

    def __exit__(self, *exc):
        for k, v in self.old.items():
            _lib.set_option(k, v)


def _flat_gaussians():
    """Flat Gaussians as a trained gs_flat checkpoint holds them: the raw (xyz, _scaling [P,3] with the log eps column,
    _rotation) of a mesh-Gaussian expansion, with its SH features and opacity logits (CPU tensors)."""
    if not _params:
        p = scenes.init_mesh_gaussians(*scenes.icosphere(4), K=3, seed=21, trained_like=True)
        with torch.no_grad():
            xyz, sl, rr = MeshGaussianModel.from_params(p, "cuda").expand_fused(activated=False)
        _params.update(xyz=xyz.cpu(), _scaling=sl.cpu(), _rotation=rr.cpu(), features_dc=p._features_dc,
                       features_rest=p._features_rest, opacity=p._opacity)
    return _params


def _model(degree=3):
    g = _flat_gaussians()
    return PointsModel.from_gaussians(g["xyz"], g["_scaling"], g["_rotation"], g["features_dc"], g["features_rest"], g["opacity"],
                                      "cuda", active_sh_degree=degree)


def _camera():
    return scenes.look_at_camera((2.2, 0.7, 1.0), (0, 0, 0), W, H)


def _render_twice(r, cam, bg, **kw):
    """(synchronising render, sync-free render) of one view, cloned."""
    first = [t.clone() for t in r.render(cam, bg, **kw)]
    second = [t.clone() for t in r.render(cam, bg, **kw)]
    torch.cuda.synchronize()
    return first, second


def _oracle(model, cam, triangles=None, scale_modifier=1.0, antialiasing=False):
    """The oracle rasterizer on the GPU's pseudo-mesh expansion of the frame's triangles, checked against the oracle's own
    (points_prepare_scaling_rot, points_get_scaling, normalised quaternion) first so that integer outputs compare bit for
    bit; opacities are the oracle's sigmoid of the logits."""
    tri = model.triangles if triangles is None else triangles
    xyz, sc, rot = (t.cpu() for t in expansion.points_prepare_scaling_rot(tri, model.eps_s0, activated=True))
    otri = tri.cpu()
    osl, orr = oexp.points_prepare_scaling_rot(otri, model.eps_s0)
    osc, orot = oexp.points_get_scaling(osl, model.eps_s0), torch.nn.functional.normalize(orr)
    assert torch.equal(xyz, otri[:, 0])
    assert bool(((sc - osc).abs() <= 1e-4 * osc + 1e-7).all()) and float((rot - orot).abs().max()) <= 1e-5
    op = torch.sigmoid(model._opacity.cpu())
    S = settings_from_camera(cam, sh_degree=model.active_sh_degree, bg=BG, scale_modifier=scale_modifier, antialiasing=antialiasing)
    return raster.forward(S, xyz, op, shs=model._features.cpu().contiguous(), scales=sc, rotations=rot)


@pytest.mark.parametrize("degree,scale_modifier,antialiasing", [(0, 1.0, False), (1, 1.0, False), (2, 1.0, False), (3, 1.0, False),
                                                                 (3, 1.3, False), (3, 1.0, True)])
def test_render_matches_the_oracle(degree, scale_modifier, antialiasing):
    model = _model(degree)
    cam = _camera()
    r = PointsRenderer(model, W, H)
    _, (image, radii, invd) = _render_twice(r, cam.to("cuda"), torch.tensor(BG, device="cuda"), scale_modifier=scale_modifier,
                                            antialiasing=antialiasing)
    st = _oracle(model, cam, scale_modifier=scale_modifier, antialiasing=antialiasing)
    np.testing.assert_array_equal(radii.cpu().numpy(), st.radii)
    assert r.last_num_rendered == st.N and r.overflows == 0
    ok = assert_image_parity(st, image.cpu().numpy())
    assert np.abs(invd.cpu().numpy() - st.invdepth)[:, ok].max() <= 1e-5


def test_hotdog_sweep_matches_the_oracle():
    """scripts/render_points_time_animated.py: every frame renders transform_hotdog(triangles, t)."""
    model = _model()
    cam = _camera()
    cam_d, bg = cam.to("cuda"), torch.tensor(BG, device="cuda")
    r = PointsRenderer(model, W, H)
    r.render(cam_d, bg)
    for t in HOTDOG_TIMES:
        tri = scenes.transform_hotdog(model.triangles, t)
        image, radii, invd = r.render(cam_d, bg, triangles=tri)
        st = _oracle(model, cam, triangles=tri)
        np.testing.assert_array_equal(radii.cpu().numpy(), st.radii)
        ok = assert_image_parity(st, image.cpu().numpy())
        assert np.abs(invd.cpu().numpy() - st.invdepth)[:, ok].max() <= 1e-5
    assert r.overflows == 0


@pytest.mark.parametrize("t", [None, *HOTDOG_TIMES])
@pytest.mark.parametrize("antialiasing", [False, True])
def test_render_is_bit_identical_to_the_shim(t, antialiasing):
    model = _model()
    cam_d, bg = _camera().to("cuda"), torch.tensor(BG, device="cuda")
    tri = None if t is None else scenes.transform_hotdog(model.triangles, t)
    r = PointsRenderer(model, W, H)
    sync, free = _render_twice(r, cam_d, bg, triangles=tri, antialiasing=antialiasing)
    with torch.no_grad():
        shim = render_points_frame(model, cam_d, bg, triangles=tri, antialiasing=antialiasing)
    for a, b, c in zip(shim, sync, free):
        assert torch.equal(a, b) and torch.equal(a, c)


@pytest.mark.parametrize("opts", FWD_OPTION_SETS, ids=_opt_id)
def test_sync_free_render_is_bit_identical_to_the_synchronising_one(opts):
    model = _model()
    cam_d, bg = _camera().to("cuda"), torch.tensor(BG, device="cuda")
    with _Options(opts):
        r = PointsRenderer(model, W, H)
        sync, free = _render_twice(r, cam_d, bg)
        N = r.last_num_rendered
    assert r.overflows == 0 and r.capacity > N > 0
    for a, b in zip(sync, free):
        assert torch.equal(a, b)


@pytest.mark.parametrize("opts", [{}, {"bin_impl": 1}], ids=_opt_id)
def test_overflowed_render_gives_the_background_then_recovers(opts):
    model = _model()
    cam_d, bg = _camera().to("cuda"), torch.tensor(BG, device="cuda")
    with _Options(opts):
        r = PointsRenderer(model, W, H)
        _, good = _render_twice(r, cam_d, bg)
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
    """gms_binning_bytes(capacity) is the region a training forward needs: the sort buffers plus four survivor lists of 4 B
    per duplicate.  The points render asks for at least those lists less; with counting binning (bin_impl=1 at this
    size), for the point list only."""
    model = _model()
    cam_d, bg = _camera().to("cuda"), torch.tensor(BG, device="cuda")
    with _Options(opts):
        r = PointsRenderer(model, W, H)
        _render_twice(r, cam_d, bg)
    cap = r.capacity
    req = r._scratch["requested"][_lib.BUF_BINNING]
    full = int(_lib.lib().gms_binning_bytes(cap, model.triangles.shape[0]))
    print(f"[points render] capacity {cap}: binning request {req} B, with survivor lists {full} B")
    assert full - req >= 16 * cap
    if opts.get("bin_impl") == 1:
        assert req <= 4 * cap + 512


def test_flat_checkpoint_loads_to_the_reference_pseudo_mesh(tmp_path, golden_dir):
    """A gs_flat point_cloud.ply (scale_0 = log eps_s0, scale_1..2 the in-plane log-scales) -> PointsModel: the triangles are
    points_prepare_vertices of the file's tensors and the reference's prepare_vertices output (points_model.npz)."""
    g = np.load(f"{golden_dir}/points_model.npz")
    P = g["pv_xyz"].shape[0]
    gen = torch.Generator().manual_seed(2)
    fdc, frest, op = torch.randn(P, 1, 3, generator=gen), torch.randn(P, 15, 3, generator=gen), torch.randn(P, 1, generator=gen)
    sl3 = torch.cat([torch.full((P, 1), math.log(1e-8)), torch.tensor(g["pv_scaling"])], dim=1)
    path = str(tmp_path / "point_cloud.ply")
    io_ply.save_gaussian_ply(path, torch.tensor(g["pv_xyz"]), fdc, frest, op, sl3, torch.tensor(g["pv_rotation"]))
    m = PointsModel.from_flat_checkpoint(path, "cuda", active_sh_degree=2)
    want = expansion.points_prepare_vertices(torch.tensor(g["pv_xyz"]).cuda(), sl3.cuda(), torch.tensor(g["pv_rotation"]).cuda())
    assert torch.equal(m.triangles, want)
    np.testing.assert_allclose(m.triangles.cpu().numpy(), g["pv_triangles"], rtol=0, atol=1e-6)
    assert torch.equal(m._features.cpu(), torch.cat([fdc, frest], dim=1)) and torch.equal(m._opacity.cpu(), op)
    assert m.active_sh_degree == 2 and m.max_sh_degree == 3 and m.eps_s0 == 1e-8


def _views(n):
    cams = [c.to("cuda") for c in scenes.ring_cameras(n, 2.6, W, H)]
    g = torch.Generator().manual_seed(5)
    gts8 = [(torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).cuda() for _ in range(n)]
    return cams, gts8


@pytest.mark.parametrize("protocol", ["training_report", "metrics"])
def test_evaluate_matches_a_per_view_loop(protocol):
    cams, gts8 = _views(6)
    gts = [io_image.to_device_float(t).clone() for t in gts8]
    bg = torch.tensor(BG, device="cuda")
    model = _model()
    res = PointsRenderer(model, W, H).evaluate(cams, gts, bg, protocol=protocol)
    assert res.per_view.shape == (6, 4) and res.rerun == []
    loop = PointsRenderer(model, W, H)
    for v, (cam, gt) in enumerate(zip(cams, gts)):
        want = image_metrics(loop.render(cam, bg)[0], gt, protocol).cpu()
        assert torch.equal(res.per_view[v].view(torch.int64), want.view(torch.int64)), (v, res.per_view[v], want)
    assert torch.equal(res.mean, res.per_view.mean(0))


def test_evaluate_u8_ground_truth_and_overflow_reruns_give_the_same_bits():
    cams, gts8 = _views(6)
    gts = [io_image.to_device_float(t).clone() for t in gts8]
    bg = torch.tensor(BG, device="cuda")
    model = _model()
    clean = PointsRenderer(model, W, H).evaluate(cams, gts, bg)
    assert clean.rerun == []
    r8 = PointsRenderer(model, W, H)
    from_u8 = r8.evaluate(cams, gts8, bg)
    assert torch.equal(from_u8.per_view.view(torch.int64), clean.per_view.view(torch.int64))
    ns = sorted(r8._view_n[r8._view_key(c)][0] for c in cams)
    assert ns[0] < ns[-1]
    r = PointsRenderer(model, W, H)
    r.capacity_override = (ns[0] + ns[-1]) // 2
    res = r.evaluate(cams, gts8, bg)
    print(f"[points evaluate] N per view {ns}, capacity {r.capacity_override}: re-ran views {res.rerun}")
    assert res.rerun and r.overflows == len(res.rerun)
    assert torch.equal(res.per_view.view(torch.int64), clean.per_view.view(torch.int64))


def test_triangles_override_leaves_the_model_untouched():
    model = _model()
    before = [t.clone() for t in (model.triangles, model._features, model._opacity)]
    cam_d, bg = _camera().to("cuda"), torch.tensor(BG, device="cuda")
    tri = scenes.transform_hotdog(model.triangles, 2.5)
    r = PointsRenderer(model, W, H)
    moved = [t.clone() for t in r.render(cam_d, bg, triangles=tri)]
    rest = r.render(cam_d, bg)[0].clone()
    torch.cuda.synchronize()
    for a, b in zip(before, (model.triangles, model._features, model._opacity)):
        assert torch.equal(a, b)
    assert not torch.equal(moved[0], rest)
    moved_model = PointsModel(tri, model._features, model._opacity, model.active_sh_degree)
    assert torch.equal(moved[0], PointsRenderer(moved_model, W, H).render(cam_d, bg)[0])
    with pytest.raises(RuntimeError):
        r.render(cam_d, bg, triangles=tri[:-1].contiguous())


def test_bad_arguments_are_refused():
    model = _model()
    r = PointsRenderer(model, W, H)
    P = model.triangles.shape[0]

    def call(**kw):
        a = _lib.PointsRenderArgs()
        a.P, a.M, a.eps = P, model._features.shape[1], model.eps_s0
        a.triangles, a.features, a.opacity_raw = model.triangles.data_ptr(), model._features.data_ptr(), model._opacity.data_ptr()
        a.settings.image_width, a.settings.image_height = W, H
        a.image, a.invdepth, a.radii = r.image.data_ptr(), r.invdepth.data_ptr(), r.radii.data_ptr()
        a.workspace, a.workspace_bytes = r.ws.data_ptr(), r.ws.numel()
        for k, v in kw.items():
            setattr(a, k, v)
        return _lib.lib().gms_points_render_frame(C.byref(a), r._cb, None, None)

    _lib.launch_count(reset=True)
    for kw in ({"triangles": None}, {"features": None}, {"opacity_raw": None}, {"image": None}, {"invdepth": None}, {"radii": None},
               {"workspace": None}, {"workspace_bytes": r.ws.numel() - 1}, {"P": -1}):
        assert call(**kw) == _lib.GMS_E_ARG, kw
        assert b"gms_points_render_frame" in _lib.lib().gms_last_error(), kw
    assert _lib.launch_count(reset=True) == 0
    assert int(_lib.lib().gms_points_render_workspace_bytes(P, W, H)) == int(_lib.lib().gms_render_workspace_bytes(P, W, H))
