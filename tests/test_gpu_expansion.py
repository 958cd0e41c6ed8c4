"""-m gpu: fused expansion kernels vs the reference-pinned oracle (oracle/expansion.py) and the golden vectors
the reference's own Python produced; plus the whole frame (expansion -> rasterizer -> loss -> backward)."""
import os

import numpy as np
import pytest
import torch

from gms_b200 import expansion, scenes
from gms_b200.model import MeshGaussianModel
from oracle import expansion as oexp
from helpers import settings_from_camera

pytestmark = pytest.mark.gpu


def test_expand_matches_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "expansion_mesh.npz"))
    dev = "cuda"
    v = torch.tensor(g["vertices"], device=dev, requires_grad=True)
    a = torch.tensor(g["_alpha"], device=dev, requires_grad=True)
    s = torch.tensor(g["_scale"], device=dev, requires_grad=True)
    f = torch.tensor(g["faces"], device=dev)
    xyz, sl, rr, alpha, tri = expansion.expand(v, f, a, s, activated=False)
    np.testing.assert_allclose(alpha.cpu().numpy(), g["alpha"], atol=1e-7)
    np.testing.assert_array_equal(tri.cpu().numpy(), g["triangles"])
    np.testing.assert_allclose(xyz.detach().cpu().numpy(), g["xyz"], atol=1e-6)
    np.testing.assert_allclose(sl.detach().cpu().numpy(), g["_scaling"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(rr.detach().cpu().numpy(), g["_rotation"], atol=1e-6)
    rot = torch.nn.functional.normalize(rr)
    loss = (xyz * torch.tensor(g["wx"], device=dev)).sum() + (sl * torch.tensor(g["ws"], device=dev)).sum() + \
           (rot * torch.tensor(g["wr"], device=dev)).sum()
    loss.backward()
    np.testing.assert_allclose(v.grad.cpu().numpy(), g["g_vertices"], rtol=3e-4, atol=3e-4)
    np.testing.assert_allclose(a.grad.cpu().numpy(), g["g_alpha"], rtol=3e-4, atol=1e-5)
    np.testing.assert_allclose(s.grad.cpu().numpy(), g["g_scale"], rtol=3e-4, atol=1e-5)
    # activated outputs
    x2, sa, ra, _, _ = expansion.expand(v.detach(), f, a.detach(), s.detach(), activated=True)
    np.testing.assert_allclose(sa.cpu().numpy(), g["get_scaling"], rtol=1e-5)
    np.testing.assert_allclose(ra.cpu().numpy(), g["get_rotation"], atol=1e-6)


@pytest.mark.parametrize("level,K", [(3, 3), (5, 5)])
def test_two_step_protocol_equals_fused_and_oracle(level, K):
    """update_alpha() + prepare_scaling_rot() (what train.py:154-157 calls) == one fused launch == oracle autograd."""
    p = scenes.init_mesh_gaussians(*scenes.icosphere(level), K=K, seed=1)
    dev = "cuda"
    m = MeshGaussianModel.from_params(p, dev)
    P = m._scale.shape[0]
    gen = torch.Generator().manual_seed(0)
    wx, ws, wr = torch.randn(P, 3, generator=gen), torch.randn(P, 3, generator=gen), torch.randn(P, 4, generator=gen)
    loss = (m.get_xyz * wx.to(dev)).sum() + (m._scaling * ws.to(dev)).sum() + (m.get_rotation * wr.to(dev)).sum()
    loss.backward()
    g2 = [t.grad.clone() for t in (m.vertices, m._alpha, m._scale)]
    for t in (m.vertices, m._alpha, m._scale):
        t.grad = None
    xyz, sl, rr = m.expand_fused(activated=False)
    loss = (xyz * wx.to(dev)).sum() + (sl * ws.to(dev)).sum() + (torch.nn.functional.normalize(rr) * wr.to(dev)).sum()
    loss.backward()
    g1 = [t.grad.clone() for t in (m.vertices, m._alpha, m._scale)]
    tv, ta, ts = (x.clone().requires_grad_(True) for x in (p.vertices, p._alpha, p._scale))
    oxyz, osl, orr, _, _ = oexp.expand(tv, p.faces, ta, ts)
    (oxyz * wx).sum().add((osl * ws).sum()).add((torch.nn.functional.normalize(orr) * wr).sum()).backward()
    np.testing.assert_allclose(xyz.detach().cpu().numpy(), oxyz.detach().numpy(), atol=2e-6)
    np.testing.assert_allclose(sl.detach().cpu().numpy(), osl.detach().numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(rr.detach().cpu().numpy(), orr.detach().numpy(), atol=2e-6)
    for a, b, c in zip(g1, g2, (tv.grad, ta.grad, ts.grad)):
        sc = c.abs().max().item()
        assert (a.cpu() - c).abs().max().item() / sc < 1e-3
        assert (b.cpu() - c).abs().max().item() / sc < 1e-3


def test_whole_frame_gradients_reach_mesh_parameters():
    """expansion -> activations -> rasterizer -> loss -> backward: gradient w.r.t. vertices/_alpha/_scale/features/opacity
    equals oracle expansion autograd chained with the oracle rasterizer backward."""
    import diff_gaussian_rasterization as dgr
    from gpu_helpers import gpu_settings
    from oracle import raster
    p = scenes.init_mesh_gaussians(*scenes.icosphere(3), K=3, seed=4)
    cam = scenes.look_at_camera((2.4, 0.8, 1.0), (0, 0, 0), 256, 192)
    S = settings_from_camera(cam, bg=(1, 1, 1))
    dev = "cuda"
    m = MeshGaussianModel.from_params(p, dev)
    xyz, sc, rot = m.expand_fused(activated=True)
    r = dgr.GaussianRasterizer(raster_settings=gpu_settings(S))
    m2d = torch.zeros_like(xyz, requires_grad=True)
    color, radii, invd = r(means3D=xyz, means2D=m2d, opacities=m.get_opacity, shs=m.get_features, scales=sc, rotations=rot)
    dC = np.random.RandomState(3).randn(3, 192, 256).astype(np.float32)
    (color * torch.tensor(dC, device=dev)).sum().backward()
    # oracle chain
    tv, ta, ts, to, tdc, trest = (x.clone().requires_grad_(True) for x in (p.vertices, p._alpha, p._scale, p._opacity, p._features_dc, p._features_rest))
    oxyz, osl, orr, _, _ = oexp.expand(tv, p.faces, ta, ts)
    osc, orot, oop, ofe = oexp.activate(osl, orr, to, tdc, trest)
    # the rasterizer oracle is fed the SAME expanded values the CUDA rasterizer saw (flat mesh Gaussians make the
    # projection ill-conditioned: 1e-7 input differences would otherwise show up as 1e-4 colour differences)
    st = raster.forward(S, xyz.detach().cpu(), oop, shs=ofe.contiguous(), scales=sc.detach().cpu(), rotations=rot.detach().cpu())
    g = raster.backward(st, dC, None)
    torch.autograd.backward([oxyz, osc, orot, oop, ofe],
                            [torch.tensor(g["dL_dmeans3D"]), torch.tensor(g["dL_dscales"]), torch.tensor(g["dL_drotations"]),
                             torch.tensor(g["dL_dopacity"]), torch.tensor(g["dL_dsh"])])
    ok = st.ambiguous == 0
    assert np.abs(color.detach().cpu().numpy() - st.color)[:, ok].max() < 1e-5
    for name, a, b in [("vertices", m.vertices.grad, tv.grad), ("_alpha", m._alpha.grad, ta.grad), ("_scale", m._scale.grad, ts.grad),
                       ("_opacity", m._opacity.grad, to.grad), ("_features_dc", m._features_dc.grad, tdc.grad),
                       ("_features_rest", m._features_rest.grad, trest.grad)]:
        sc_ = b.abs().max().item() + 1e-20
        err = (a.cpu() - b).abs().max().item() / sc_
        assert err < 2e-3, f"{name}: {err:.3e}"


def test_multi_mesh_matches_reference_golden_and_merged_path(golden_dir):
    """gs_multi_mesh: per-mesh loop + cat (heterogeneous K) against the reference's GaussianMultiMeshModel output; and the
    merged single-launch path (equal K) against the per-mesh loop."""
    from gms_b200.model import MultiMeshGaussianModel
    g = np.load(os.path.join(golden_dir, "expansion_multi.npz"))
    n = int(g["n_mesh"])
    dev = "cuda"
    vs = [torch.tensor(g[f"vertices{k}"], device=dev) for k in range(n)]
    fs = [torch.tensor(g[f"faces{k}"], device=dev) for k in range(n)]
    als = [torch.tensor(g[f"_alpha{k}"], device=dev) for k in range(n)]
    scs = [torch.tensor(g[f"_scale{k}"], device=dev) for k in range(n)]
    xyz, sl, rr = MultiMeshGaussianModel.expand_per_mesh(vs, fs, als, scs)
    np.testing.assert_allclose(xyz.cpu().numpy(), g["xyz"], atol=1e-6)
    np.testing.assert_allclose(sl.cpu().numpy(), g["_scaling"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(rr.cpu().numpy(), g["_rotation"], atol=1e-6)
    # merged fast path (same K): identical to the loop
    plist = [scenes.init_mesh_gaussians(*scenes.icosphere(2, radius=0.4 + 0.2 * k), K=3, seed=k) for k in range(3)]
    for k, p in enumerate(plist):
        p.vertices += torch.tensor([1.2 * k, 0.0, 0.0])
    m = MultiMeshGaussianModel.from_mesh_params(plist, dev)
    x1, s1, r1 = m.expand_fused(activated=False)
    x2, s2, r2 = MultiMeshGaussianModel.expand_per_mesh([p.vertices.to(dev) for p in plist], [p.faces.to(dev) for p in plist],
                                                        [p._alpha.to(dev) for p in plist], [p._scale.to(dev) for p in plist])
    assert torch.equal(x1, x2) and torch.equal(s1, s2) and torch.equal(r1, r2)


def test_animated_path_reexpands_from_triangles():
    """renderer/gaussian_animated_renderer/__init__.py:61-73: xyz = alpha @ triangles and prepare_scaling_rot() from the
    TRANSFORMED triangles; our two-step ops follow the moved vertices exactly like the oracle."""
    p = scenes.init_mesh_gaussians(*scenes.icosphere(3), K=4, seed=9)
    dev = "cuda"
    m = MeshGaussianModel.from_params(p, dev)
    v_new = scenes.transform_hotdog_fly(p.vertices, 7.5)
    tri = v_new[p.faces].to(dev)
    m.triangles = tri
    m.prepare_scaling_rot()
    xyz = torch.matmul(m.alpha, tri).reshape(-1, 3)
    oxyz, osl, orr, _, _ = oexp.expand(v_new, p.faces, p._alpha, p._scale)
    np.testing.assert_allclose(xyz.detach().cpu().numpy(), oxyz.numpy(), atol=2e-6)
    np.testing.assert_allclose(m._scaling.detach().cpu().numpy(), osl.numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(m._rotation.detach().cpu().numpy(), orr.numpy(), atol=2e-6)


def test_points_pseudomesh_path_matches_reference_golden(golden_dir):
    """gs_points (renderer/gaussian_points_animated_renderer/__init__.py:61-66): triangles -> xyz / scaling / rotation."""
    g = np.load(os.path.join(golden_dir, "points_model.npz"))
    tri = torch.tensor(g["triangles"], device="cuda")
    xyz, sl, rr = expansion.points_prepare_scaling_rot(tri, activated=False)
    assert torch.equal(xyz, tri[:, 0])
    np.testing.assert_allclose(sl.cpu().numpy(), g["_scaling"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(rr.cpu().numpy(), g["_rotation"], atol=2e-6)
    _, sa, ra = expansion.points_prepare_scaling_rot(tri, activated=True)
    # s3 = (v3 - v1) . r3 is a cancellation result for near-collinear triangles: FMA contraction on the GPU moves it by ~1e-7 abs
    np.testing.assert_allclose(sa.cpu().numpy(), g["get_scaling"], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(ra.cpu().numpy(), g["get_rotation"], atol=2e-6)


def test_points_prepare_vertices_matches_golden_and_oracle(golden_dir):
    """gs_points prepare_vertices (games/flat_splatting/scene/points_gaussian_model.py:28-59) on the GPU: reference golden
    vector, the oracle on a larger random state, and the patched-model round trip prepare_vertices -> prepare_scaling_rot."""
    from oracle import expansion as oexp
    g = np.load(os.path.join(golden_dir, "points_model.npz"))
    tri = expansion.points_prepare_vertices(torch.tensor(g["pv_xyz"], device="cuda"),
                                            torch.tensor(g["pv_scaling"], device="cuda"),
                                            torch.tensor(g["pv_rotation"], device="cuda"))
    np.testing.assert_allclose(tri.cpu().numpy(), g["pv_triangles"], rtol=0, atol=1e-6)
    gen = torch.Generator().manual_seed(3)
    P = 50_001
    xyz = torch.randn(P, 3, generator=gen); sl = -3.0 + torch.randn(P, 3, generator=gen)
    q = torch.randn(P, 4, generator=gen) * 3.0
    want = oexp.points_prepare_vertices(xyz, sl, q)
    got = expansion.points_prepare_vertices(xyz.cuda(), sl.cuda(), q.cuda())
    np.testing.assert_allclose(got.cpu().numpy(), want.numpy(), rtol=0, atol=2e-6)

    class _PM:            # the attributes the reference's PointsGaussianModel methods touch
        pass
    m = _PM(); m._xyz, m._scaling, m._rotation = xyz.cuda(), sl.cuda(), q.cuda()
    expansion.patch_points_model(m)
    m.prepare_vertices()
    assert torch.equal(m.triangles, got) and torch.equal(m.v1, m._xyz)
    m.prepare_scaling_rot()
    osl, _ = oexp.points_prepare_scaling_rot(want)
    np.testing.assert_allclose(m._scaling.cpu().numpy(), osl.numpy(), rtol=0, atol=1e-4)
    longer_first = torch.sort(sl[:, 1:], dim=1, descending=True).values
    np.testing.assert_allclose(m._scaling.cpu().numpy(), longer_first.numpy(), atol=1e-4)


@pytest.mark.parametrize("level,K", [(2, 1), (3, 3), (3, 7), (1, 40)])
def test_staged_and_direct_expansion_kernels_vs_oracle(level, K):
    """The per-thread kernels the call's K selects against the oracle: at K = 1 and 3 the forward's per-Gaussian rows (17
    floats each here) fit the 48 KB staging limit and run the staged forward, at K = 7 and 40 they do not and run the direct
    one.  F is not a multiple of the 128-face block.  Outputs, and the gradients of a backward through the raw and the
    activated outputs."""
    p = scenes.init_mesh_gaussians(*scenes.icosphere(level), K=K, seed=4)
    gen = torch.Generator().manual_seed(1)
    m = MeshGaussianModel.from_params(p, "cuda")
    P = m._scale.shape[0]
    w = [torch.randn(P, c, generator=gen).cuda() for c in (3, 3, 4)]
    outs = []
    for activated in (False, True):
        xyz, sc, rot = m.expand_fused(activated=activated)
        ((xyz * w[0]).sum() + (sc * w[1]).sum() + (rot * w[2]).sum()).backward()
        outs += [xyz.detach(), sc.detach(), rot.detach()]
    tv, ta, ts = (x.clone().requires_grad_(True) for x in (p.vertices, p._alpha, p._scale))
    oxyz, osl, orr, _, _ = oexp.expand(tv, p.faces, ta, ts)
    ow = [t.cpu() for t in w]
    loss = (oxyz * ow[0]).sum() + (osl * ow[1]).sum() + (orr * ow[2]).sum()
    (loss + (oxyz * ow[0]).sum() + (torch.exp(osl) * ow[1]).sum() + (torch.nn.functional.normalize(orr) * ow[2]).sum()).backward()
    np.testing.assert_allclose(outs[0].cpu().numpy(), oxyz.detach().numpy(), atol=1e-6)
    np.testing.assert_allclose(outs[1].cpu().numpy(), osl.detach().numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(outs[2].cpu().numpy(), orr.detach().numpy(), atol=2e-6)
    for a, c in zip((m.vertices.grad, m._alpha.grad, m._scale.grad), (tv.grad, ta.grad, ts.grad)):
        assert (a.cpu() - c).abs().max().item() / c.abs().max().item() < 1e-3
