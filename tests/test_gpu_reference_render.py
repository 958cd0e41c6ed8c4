"""-m gpu: the reference's rendering protocol on the GPU on top of the drop-in module, against the oracle.

The reference's GaussianMeshModel expands a mesh with PyTorch ops (update_alpha / prepare_scaling_rot,
games/mesh_splatting/scene/gaussian_mesh_model.py:86-169) and its renderers hand the model's getters to
`diff_gaussian_rasterization` (renderer/gaussian_renderer/__init__.py:25-111, renderer/gaussian_animated_renderer/__init__.py:21-121).
Here the "stock" model is that PyTorch expansion as oracle/expansion.py restates it (pinned to the reference by
tests/test_oracle_golden.py), run on the GPU; the "patched" model swaps the fused kernels in with expansion.patch_mesh_model().
tests/golden/reference_render.npz holds what the reference's own code computed for these scenes (a seeded sample of the
Gaussians; tests/golden/make_reference_render_golden.py), and images + gradients are compared with the oracle chain
(oracle/expansion.py -> oracle/gms_oracle.c).

What is not exercised any more: the reference's own code itself.  The stock model is built directly from the scene
parameters, not through GaussianMeshModel.create_from_pcd, and the stock-expansion render compares the oracle's expansion
with itself on the expansion side; its link to the reference is the sampled golden rows checked in
test_patched_and_stock_expansion_agree_on_the_gpu, test_reference_animated_renderer_matches_oracle and the checkpoint test."""
import math
import os
import sys

import numpy as np
import pytest
import torch

from gms_b200 import expansion, scenes
from gpu_helpers import GRAD_TOL, oracle_chain
from helpers import settings_from_camera
from oracle import expansion as oexp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_reference_render_golden import alpha_upstream, sample_rows  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "reference_render.npz"))


class StockMeshModel:
    """The attribute surface of the reference's GaussianMeshModel (gaussian_mesh_model.py:27-169 + the getters of
    scene/gaussian_model.py:95-118), expanding with the PyTorch ops of oracle/expansion.py on the model's device."""

    def __init__(self, p, device="cuda"):
        mk = lambda t: torch.nn.Parameter(t.to(device).float().clone())
        self.vertices, self._alpha, self._scale = mk(p.vertices), mk(p._alpha), mk(p._scale)
        self._opacity, self._features_dc, self._features_rest = mk(p._opacity), mk(p._features_dc), mk(p._features_rest)
        self.faces = p.faces.to(device)
        self.eps_s0 = oexp.EPS_S0
        self.active_sh_degree = self.max_sh_degree = 3

    def update_alpha(self):
        self.alpha, self.triangles, self._xyz = oexp.update_alpha(self._alpha, self.vertices, self.faces)

    def prepare_scaling_rot(self):
        self._scaling, self._rotation = oexp.prepare_scaling_rot(self.triangles, self._scale, self._alpha.shape[1], self.eps_s0)

    get_xyz = property(lambda self: self._xyz)
    get_scaling = property(lambda self: torch.exp(self._scaling))
    get_rotation = property(lambda self: torch.nn.functional.normalize(self._rotation))
    get_opacity = property(lambda self: torch.sigmoid(self._opacity))
    get_features = property(lambda self: torch.cat((self._features_dc, self._features_rest), dim=1))


def _reference_model(p):
    m = StockMeshModel(p)
    m.update_alpha(); m.prepare_scaling_rot()
    return m


def render(cam, pc, bg, triangles=None):
    """renderer/gaussian_renderer/__init__.py:25-111 (triangles=None) and renderer/gaussian_animated_renderer/__init__.py:21-121
    as the reference calls the rasterizer: its settings, its screen-space point tensor, its getters."""
    import diff_gaussian_rasterization as dgr
    screenspace_points = torch.zeros_like(pc.get_xyz, requires_grad=True, device="cuda") + 0
    if screenspace_points.requires_grad:          # not under no_grad (the reference wraps this call in try/except)
        screenspace_points.retain_grad()
    rs = dgr.GaussianRasterizationSettings(
        image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=math.tan(cam.FoVx * 0.5),
        tanfovy=math.tan(cam.FoVy * 0.5), bg=bg, scale_modifier=1.0, viewmatrix=cam.world_view_transform,
        projmatrix=cam.full_proj_transform, sh_degree=pc.active_sh_degree, campos=cam.camera_center, prefiltered=False,
        debug=False, antialiasing=False)
    means3D = pc.get_xyz
    if triangles is not None:
        means3D = torch.matmul(pc.alpha, triangles).reshape(-1, 3)
        pc.triangles = triangles
        pc.prepare_scaling_rot()
    img, radii, depth = dgr.GaussianRasterizer(raster_settings=rs)(
        means3D=means3D, means2D=screenspace_points, shs=pc.get_features, colors_precomp=None, opacities=pc.get_opacity,
        scales=pc.get_scaling, rotations=pc.get_rotation, cov3D_precomp=None)
    return {"render": img, "viewspace_points": screenspace_points, "visibility_filter": radii > 0, "radii": radii, "depth": depth}


def _assert_sample(got, ref, atol, rtol=0.0, what=""):
    got = got.detach().float().cpu().numpy()
    np.testing.assert_allclose(got[sample_rows(got.shape[0])], ref, rtol=rtol, atol=atol, err_msg=what)


def _check_against_oracle(pkg, model, st, ograds, tag, grad_tol):
    img = pkg["render"].detach().cpu().numpy()
    ok = st.ambiguous == 0
    nb = int((~ok).sum())
    err = float(np.abs(img - st.color)[:, ok].max())
    print(f"[{tag}] P={st.radii.shape[0]} N={st.N} threshold-ambiguous pixels={nb} max|image-oracle| (others)={err:.2e}")
    np.testing.assert_array_equal(pkg["radii"].cpu().numpy(), st.radii)
    assert err <= 1e-5, err
    assert nb <= 1e-3 * ok.size
    for k, ref_g in ograds.items():
        got = getattr(model, k).grad
        assert got is not None, k
        scale = max(float(ref_g.abs().max()), 1e-20)
        e = float((got.detach().cpu().reshape(ref_g.shape) - ref_g).abs().max()) / scale
        print(f"[{tag}] grad {k}: max err / max|ref| = {e:.2e}")
        assert e <= grad_tol.get(k, 2e-4), (k, e)


@pytest.mark.parametrize("patched", [False, True])
def test_reference_render_on_stock_mesh_model_matches_oracle(patched):
    p = scenes.init_mesh_gaussians(*scenes.icosphere(3), K=3, seed=11, trained_like=True)
    cam = scenes.look_at_camera((2.3, 0.9, 1.1), (0, 0, 0), 400, 304)
    m = _reference_model(p)
    if patched:
        expansion.patch_mesh_model(m)
        m.update_alpha(); m.prepare_scaling_rot()      # train.py:154-157
    bg = torch.ones(3, device="cuda")
    pkg = render(cam.to("cuda"), m, bg)
    rs = np.random.RandomState(3)
    dC = (rs.randn(3, cam.image_height, cam.image_width) / (cam.image_width * cam.image_height)).astype(np.float32)
    (pkg["render"] * torch.tensor(dC, device="cuda")).sum().backward()
    assert pkg["viewspace_points"].grad is not None and pkg["visibility_filter"].dtype == torch.bool
    S = settings_from_camera(cam, bg=(1, 1, 1))
    st, og = oracle_chain(p, S, dC, (m.get_xyz, m.get_scaling, m.get_rotation))
    _check_against_oracle(pkg, m, st, og, f"render/{'patched' if patched else 'stock'}-expansion", GRAD_TOL)


def test_patched_and_stock_expansion_agree_on_the_gpu(golden):
    p = scenes.init_mesh_gaussians(*scenes.icosphere(3), K=5, seed=12, trained_like=True)
    a = _reference_model(p)
    b = expansion.patch_mesh_model(_reference_model(p))
    b.update_alpha(); b.prepare_scaling_rot()
    for k, tol in (("alpha", 1e-6), ("triangles", 0.0), ("_xyz", 1e-6), ("_scaling", 1e-5), ("_rotation", 2e-6)):
        x, y = getattr(a, k).detach(), getattr(b, k).detach()
        assert x.shape == y.shape and float((x - y).abs().max()) <= tol, k
    # ... and both agree with what the reference's own GaussianMeshModel computed for this mesh
    assert float(b.triangles.detach().double().sum()) == float(golden["exp_triangles_sum"])
    for k, ref, tol in (("alpha", "exp_alpha", 1e-6), ("_xyz", "exp_xyz", 2e-6), ("_scaling", "exp_scaling", 1e-5),
                        ("_rotation", "exp_rotation", 2e-6)):
        for m in (a, b):
            x = getattr(m, k)
            _assert_sample(x.reshape(-1, x.shape[-1]), golden[ref], tol, what=k)
    # alpha stays differentiable on the patched model (renderer/gaussian_animated_renderer/__init__.py:61-64 consumes it)
    F, K = p._alpha.shape[:2]
    g = torch.tensor(alpha_upstream(F, K), device="cuda")
    (b.alpha * g).sum().backward()
    (a.alpha * g).sum().backward()
    scale = float(golden["exp_alpha_grad_absmax"])
    assert float((a._alpha.grad - b._alpha.grad).abs().max()) <= 1e-5 * float(a._alpha.grad.abs().max())
    _assert_sample(b._alpha.grad.reshape(-1, 3), golden["exp_alpha_grad"], 1e-5 * scale, what="_alpha.grad")


@pytest.mark.parametrize("t", [0.0, 2.1, 5.7])
def test_reference_animated_renderer_matches_oracle(golden, t):
    """scripts/render_time_animated.py:68-87: vertices moved by transform_hotdog_fly(t), triangles gathered, and
    gaussian_animated_renderer.render(idxs, triangles, ...) re-expanding from them -- here with gradients as well."""
    p = scenes.init_mesh_gaussians(*scenes.icosphere(3), K=3, seed=13, trained_like=True)
    cam = scenes.look_at_camera((2.6, -0.7, 0.8), (0, 0, 0), 368, 272)
    m = expansion.patch_mesh_model(_reference_model(p))
    m.update_alpha(); m.prepare_scaling_rot()
    new_v = scenes.transform_hotdog_fly(p.vertices, t)
    tri = new_v[p.faces]
    bg = torch.ones(3, device="cuda")
    pkg = render(cam.to("cuda"), m, bg, triangles=tri.cuda())
    rs = np.random.RandomState(4)
    dC = (rs.randn(3, cam.image_height, cam.image_width) / (cam.image_width * cam.image_height)).astype(np.float32)
    (pkg["render"] * torch.tensor(dC, device="cuda")).sum().backward()
    S = settings_from_camera(cam, bg=(1, 1, 1))
    with torch.no_grad():
        means3D = torch.matmul(m.alpha, tri.cuda()).reshape(-1, 3)     # the renderer's own expression (:61-67)
    tag = f"anim_{t:.1f}"
    _assert_sample(means3D, golden[tag + "_means3D"], 2e-6, what="means3D")
    _assert_sample(m.get_scaling, golden[tag + "_scales"], 0.0, 1e-5, what="scales")
    _assert_sample(m.get_rotation, golden[tag + "_rotations"], 4e-6, what="rotations")
    st, og = oracle_chain(p, S, dC, (means3D, m.get_scaling, m.get_rotation), triangles=tri)
    og.pop("vertices")                      # the animated path feeds triangles directly: no gradient reaches pc.vertices
    _check_against_oracle(pkg, m, st, og, f"animated t={t}", GRAD_TOL)


def test_checkpoint_written_here_loads_in_the_reference(golden, tmp_path):
    """io_ply.save_mesh_model writes what the reference's own GaussianMeshModel.load_ply (gaussian_mesh_model.py:211-225 ->
    scene/gaussian_model.py:226-262) read back from the same model's checkpoint (the fixture), and the reference's
    render() of that checkpoint gives the same image as the model that was saved."""
    from gms_b200 import io_ply
    from gms_b200.model import MeshGaussianModel
    from gms_b200.trainer import render_frame

    p = scenes.init_mesh_gaussians(*scenes.icosphere(3), K=3, seed=31, trained_like=True)
    ours = MeshGaussianModel.from_params(p, "cuda")
    ply = str(tmp_path / "point_cloud" / "iteration_30000" / "point_cloud.ply")
    io_ply.save_mesh_model(ply, ours)
    g = io_ply.load_gaussian_ply(ply)
    params = torch.load(ply.replace("point_cloud.ply", "model_params.pt"), weights_only=False)
    assert params["vertices"].is_cuda and params["_alpha"].is_cuda and params["faces"].is_cuda   # load_ply uses them where they are
    _assert_sample(g["_xyz"], golden["ckpt_ply_xyz"], 2e-6, what="ply xyz")
    _assert_sample(g["_opacity"], golden["ckpt_opacity"], 0.0, what="opacity")
    for k, ref in (("_features_dc", "ckpt_features_dc"), ("_features_rest", "ckpt_features_rest")):
        got = g[k].numpy()
        np.testing.assert_array_equal(got[sample_rows(got.shape[0])], golden[ref], err_msg=k)
    np.testing.assert_array_equal(params["vertices"].detach().cpu().numpy(), golden["ckpt_vertices"])
    assert int(params["faces"].sum()) == int(golden["ckpt_faces_sum"])
    _assert_sample(params["_alpha"].reshape(-1, 3), golden["ckpt_alpha"], 0.0, what="_alpha")
    _assert_sample(params["_scale"], golden["ckpt_scale"], 0.0, what="_scale")

    m = _reference_model(io_ply.load_mesh_model(ply))
    _assert_sample(m.get_xyz, golden["ckpt_xyz"], 2e-6, what="xyz")
    _assert_sample(m.get_scaling, golden["ckpt_scales"], 0.0, 1e-5, what="scales")
    _assert_sample(m.get_rotation, golden["ckpt_rotations"], 4e-6, what="rotations")
    cam = scenes.look_at_camera((2.3, 0.9, 1.1), (0, 0, 0), 320, 240).to("cuda")
    bg = torch.ones(3, device="cuda")
    with torch.no_grad():
        a = render(cam, m, bg)["render"]
        b = render_frame(ours, cam, bg, fused=False)[0]
    # the reference's PyTorch expansion and the fused kernels agree to ~1e-7 on the Gaussians, so the two images agree to
    # 1e-5 except where a 1/255 blending threshold flips (a handful of pixels, each by at most one splat's contribution)
    err = (a - b).abs().amax(dim=0)
    assert float((err > 1e-5).float().mean()) <= 1e-3 and float(err.max()) <= 2e-2, (float((err > 1e-5).float().mean()), float(err.max()))
