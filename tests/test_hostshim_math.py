"""The product's per-element maths (csrc/gms_preprocess.cuh, csrc/gms_expand.cuh -- the SAME functions the
CUDA kernels call per thread) compiled for the CPU and checked against the oracle.  No GPU needed; the warp-level
composite kernels are covered by the -m gpu tests."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from gms_b200 import _lib, scenes
from oracle import expansion as oexp
from oracle import preprocess64, raster
from preprocess_budget_cases import check_per_element
from helpers import settings_from_camera, random_gaussians
from hostshim import build_shim


@pytest.fixture(scope="module")
def shim():
    return C.CDLL(build_shim.build())


def _np(t):
    return np.ascontiguousarray(t.detach().cpu().numpy() if hasattr(t, "detach") else t)


def _ptr(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _expand_args(V, F, K, vertices, faces, tri_in, alpha_raw, scale_raw, eps, **outs):
    a = _lib.ExpandArgs()
    a.V, a.F, a.K = V, F, K
    a.vertices, a.faces, a.triangles_in = [None if x is None else x.ctypes.data for x in (vertices, faces, tri_in)]
    a.alpha_raw, a.scale_raw, a.eps = alpha_raw.ctypes.data, scale_raw.ctypes.data, eps
    for k, v in outs.items():
        setattr(a, k, None if v is None else v.ctypes.data)
    return a


def _mesh_case(golden_dir):
    g = np.load(os.path.join(golden_dir, "expansion_mesh.npz"))
    return g, g["vertices"].astype(np.float32), g["faces"].astype(np.int64), g["_alpha"].astype(np.float32), g["_scale"].astype(np.float32)


def test_expand_forward_matches_reference_golden(shim, golden_dir):
    g, v, f, a, s = _mesh_case(golden_dir)
    F, K = a.shape[:2]; P = F * K
    alpha = np.zeros((F, K, 3), np.float32); tri = np.zeros((F, 3, 3), np.float32); xyz = np.zeros((P, 3), np.float32)
    sl = np.zeros((P, 3), np.float32); rr = np.zeros((P, 4), np.float32); sa = np.zeros((P, 3), np.float32); ra = np.zeros((P, 4), np.float32)
    args = _expand_args(v.shape[0], F, K, v, f, None, a, s, 1e-8, alpha=alpha, triangles=tri, xyz=xyz, scaling_log=sl,
                        rotation_raw=rr, scaling_act=sa, rotation_act=ra)
    assert shim.shim_expand_forward(C.byref(args)) == 0
    np.testing.assert_allclose(alpha, g["alpha"], atol=1e-7)
    np.testing.assert_array_equal(tri, g["triangles"])
    np.testing.assert_allclose(xyz, g["xyz"], atol=1e-6)
    np.testing.assert_allclose(sl, g["_scaling"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(rr, g["_rotation"], atol=1e-6)
    np.testing.assert_allclose(sa, g["get_scaling"], rtol=1e-5)
    np.testing.assert_allclose(ra, g["get_rotation"], atol=1e-6)


def test_expand_backward_matches_reference_autograd(shim, golden_dir):
    g, v, f, a, s = _mesh_case(golden_dir)
    F, K = a.shape[:2]; P = F * K
    args = _expand_args(v.shape[0], F, K, v, f, None, a, s, 1e-8)
    gr = _lib.ExpandGrads()
    wx, ws, wr = [np.ascontiguousarray(g[k], np.float32) for k in ("wx", "ws", "wr")]
    dv = np.zeros_like(v); da = np.zeros_like(a); ds = np.zeros_like(s)
    # golden loss = <xyz,wx> + <_scaling,ws> + <normalize(_rotation),wr>
    gr.dL_dxyz, gr.dL_dscaling_log, gr.dL_drotation_act = wx.ctypes.data, ws.ctypes.data, wr.ctypes.data
    gr.dL_dvertices, gr.dL_dalpha_raw, gr.dL_dscale_raw = dv.ctypes.data, da.ctypes.data, ds.ctypes.data
    assert shim.shim_expand_backward(C.byref(args), C.byref(gr)) == 0
    np.testing.assert_allclose(dv, g["g_vertices"], rtol=2e-4, atol=2e-4)
    np.testing.assert_allclose(da, g["g_alpha"], rtol=2e-4, atol=1e-5)
    np.testing.assert_allclose(ds, g["g_scale"], rtol=2e-4, atol=1e-5)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_expand_backward_random_vs_oracle_autograd(shim, seed):
    """Random meshes / random upstream gradients on every output, incl. exp-activated scaling and raw rotation."""
    rs = np.random.RandomState(seed)
    v, f = scenes.icosphere(2)
    v = (v * (1 + 0.2 * rs.randn(*v.shape))).astype(np.float32)
    F, K = f.shape[0], 2 + seed
    P = F * K
    a = rs.rand(F, K, 3).astype(np.float32); s = (0.3 + rs.rand(P, 1)).astype(np.float32)
    wx, wsl, wrr, wsa, wra = [rs.randn(P, d).astype(np.float32) for d in (3, 3, 4, 3, 4)]
    wsa[:, 0] = 0   # exp(_scaling)[:,0] ~ 2e-8: its gradient path is numerically meaningless (SURVEY section 7)
    tv = torch.tensor(v, requires_grad=True); ta = torch.tensor(a, requires_grad=True); ts = torch.tensor(s, requires_grad=True)
    xyz, sl, rr, _, _ = oexp.expand(tv, torch.tensor(f), ta, ts)
    loss = (xyz * torch.tensor(wx)).sum() + (sl * torch.tensor(wsl)).sum() + (rr * torch.tensor(wrr)).sum() + \
           (torch.exp(sl) * torch.tensor(wsa)).sum() + (torch.nn.functional.normalize(rr) * torch.tensor(wra)).sum()
    loss.backward()
    args = _expand_args(v.shape[0], F, K, v, f, None, a, s, 1e-8)
    gr = _lib.ExpandGrads()
    dv = np.zeros_like(v); da = np.zeros_like(a); ds = np.zeros_like(s)
    gr.dL_dxyz, gr.dL_dscaling_log, gr.dL_drotation_raw, gr.dL_dscaling_act, gr.dL_drotation_act = [x.ctypes.data for x in (wx, wsl, wrr, wsa, wra)]
    gr.dL_dvertices, gr.dL_dalpha_raw, gr.dL_dscale_raw = dv.ctypes.data, da.ctypes.data, ds.ctypes.data
    assert shim.shim_expand_backward(C.byref(args), C.byref(gr)) == 0
    sc = np.abs(tv.grad.numpy()).max()
    assert np.abs(dv - tv.grad.numpy()).max() / sc < 5e-4
    np.testing.assert_allclose(da, ta.grad.numpy(), rtol=1e-3, atol=1e-4 * np.abs(ta.grad.numpy()).max())
    np.testing.assert_allclose(ds, ts.grad.numpy(), rtol=1e-3, atol=1e-4 * np.abs(ts.grad.numpy()).max())


def test_expand_triangles_in_path(shim):
    """Animated path: triangles handed in directly (gaussian_animated_renderer:61-73); dL_dtriangles written."""
    rs = np.random.RandomState(5)
    v, f = scenes.icosphere(1)
    tri = v[f].astype(np.float32)
    F, K = f.shape[0], 2; P = F * K
    a = rs.rand(F, K, 3).astype(np.float32); s = np.ones((P, 1), np.float32)
    xyz = np.zeros((P, 3), np.float32); sl = np.zeros((P, 3), np.float32); rr = np.zeros((P, 4), np.float32)
    args = _expand_args(0, F, K, None, None, tri, a, s, 1e-8, xyz=xyz, scaling_log=sl, rotation_raw=rr)
    assert shim.shim_expand_forward(C.byref(args)) == 0
    x2, sl2, rr2, _, _ = oexp.expand(torch.tensor(v), torch.tensor(f), torch.tensor(a), torch.tensor(s))
    np.testing.assert_allclose(xyz, x2.numpy(), atol=1e-6)
    np.testing.assert_allclose(sl, sl2.numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(rr, rr2.numpy(), atol=1e-6)


def _run_pre(shim, S, g, P, M, aa=0):
    st = raster.preprocess(S, g["means3D"], g["opacities"], shs=g.get("shs"), colors_precomp=g.get("colors_precomp"),
                           scales=g.get("scales"), rotations=g.get("rotations"), cov3D_precomp=g.get("cov3D_precomp"))
    f = lambda k: None if g.get(k) is None else np.ascontiguousarray(_np(g[k]), np.float32)
    means, sc, rt, cv, op, shs, col = f("means3D"), f("scales"), f("rotations"), f("cov3D_precomp"), f("opacities"), f("shs"), f("colors_precomp")
    view = np.ascontiguousarray(S.viewmatrix, np.float32).reshape(16); proj = np.ascontiguousarray(S.projmatrix, np.float32).reshape(16)
    campos = np.ascontiguousarray(S.campos, np.float32)
    out = dict(radii=np.zeros(P, np.int32), means2D=np.zeros((P, 2), np.float32), depths=np.zeros(P, np.float32),
               cov3D=np.zeros((P, 6), np.float32), conic_opacity=np.zeros((P, 4), np.float32), rgb=np.zeros((P, 3), np.float32),
               clamped=np.zeros((P, 3), np.uint8), tiles=np.zeros(P, np.uint32))
    rc = shim.shim_preprocess_forward(P, S.sh_degree, M, S.image_width, S.image_height, C.c_float(S.tanfovx), C.c_float(S.tanfovy),
                                      C.c_float(S.scale_modifier), aa, _ptr(means), _ptr(sc), _ptr(rt), _ptr(cv), _ptr(op),
                                      _ptr(shs), _ptr(col), _ptr(view), _ptr(proj), _ptr(campos), _ptr(out["radii"]),
                                      _ptr(out["means2D"]), _ptr(out["depths"]), _ptr(out["cov3D"]), _ptr(out["conic_opacity"]),
                                      _ptr(out["rgb"]), _ptr(out["clamped"]), _ptr(out["tiles"]))
    assert rc == 0
    return st, out, (means, sc, rt, cv, op, shs, col, view, proj, campos)


@pytest.mark.parametrize("aa", [0, 1])
def test_preprocess_forward_bit_exact_vs_oracle(shim, aa):
    cam = scenes.look_at_camera((2.2, 1.5, 0.9), (0, 0, 0), 320, 208)
    S = settings_from_camera(cam, antialiasing=bool(aa), scale_modifier=0.9)
    P = 4000
    g = random_gaussians(P, seed=3, extent=2.5, scale_mu=-2.5)   # extent 2.5: many culled / off-screen / straddling
    st, out, _ = _run_pre(shim, S, g, P, 16, aa)
    assert 0.2 < (st.radii > 0).mean() < 0.95
    # integer outputs and everything feeding the sort key: bit-exact
    np.testing.assert_array_equal(out["radii"], st.radii)
    np.testing.assert_array_equal(out["tiles"], st.tiles_touched)
    np.testing.assert_array_equal(out["depths"].view(np.uint32), st.depths.view(np.uint32))
    np.testing.assert_array_equal(out["means2D"].view(np.uint32), st.means2D.view(np.uint32))
    vis = st.radii > 0   # the oracle also stores cov3D for splats it later drops (empty rect); compare visible rows
    np.testing.assert_array_equal(out["cov3D"].view(np.uint32)[vis], st.cov3Ds.view(np.uint32)[vis])
    np.testing.assert_array_equal(out["conic_opacity"].view(np.uint32), st.conic_opacity.view(np.uint32))
    np.testing.assert_array_equal(out["clamped"], st.clamped)
    np.testing.assert_allclose(out["rgb"], st.rgb, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("aa", [0, 1])
def test_preprocess_backward_vs_oracle(shim, aa):
    cam = scenes.look_at_camera((2.2, 1.5, 0.9), (0, 0, 0), 160, 112)
    S = settings_from_camera(cam, antialiasing=bool(aa), scale_modifier=1.2)
    P = 1500
    g = random_gaussians(P, seed=4, extent=1.5, scale_mu=-2.3)
    st, out, (means, sc, rt, cv, op, shs, col, view, proj, campos) = _run_pre(shim, S, g, P, 16, aa)
    rs = np.random.RandomState(0)
    gin = dict(dL_dmean2D=rs.randn(P, 2), dL_dconic=rs.randn(P, 3), dL_dopacity=rs.randn(P), dL_dcolor=rs.randn(P, 3), dL_dinvdepth=rs.randn(P))
    ref = raster.preprocess_backward(st, gin)
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    d2, dc, dop, dcol, dinv = map(f32, (gin["dL_dmean2D"], gin["dL_dconic"], gin["dL_dopacity"], gin["dL_dcolor"], gin["dL_dinvdepth"]))
    o = dict(dm=np.zeros((P, 3), np.float32), dcov=np.zeros((P, 6), np.float32), dsh=np.zeros((P, 16, 3), np.float32),
             dsc=np.zeros((P, 3), np.float32), drot=np.zeros((P, 4), np.float32), dop=np.zeros(P, np.float32))
    rc = shim.shim_preprocess_backward(P, S.sh_degree, 16, S.image_width, S.image_height, C.c_float(S.tanfovx), C.c_float(S.tanfovy),
                                       C.c_float(S.scale_modifier), aa, _ptr(out["radii"]), _ptr(means), _ptr(sc), _ptr(rt), _ptr(op),
                                       _ptr(shs), _ptr(view), _ptr(proj), _ptr(campos), _ptr(out["cov3D"]), _ptr(out["clamped"]),
                                       _ptr(d2), _ptr(dc), _ptr(dop), _ptr(dcol), _ptr(dinv), _ptr(o["dm"]), _ptr(o["dcov"]),
                                       _ptr(o["dsh"]), _ptr(o["dsc"]), _ptr(o["drot"]), _ptr(o["dop"]))
    assert rc == 0
    def close(a, b, name):
        scale = np.abs(b).max()
        assert np.abs(a - b).max() <= 2e-5 * scale + 1e-12, name
    close(o["dm"], ref["dL_dmeans3D"], "means3D"); close(o["dcov"], ref["dL_dcov3D"], "cov3D")
    close(o["dsh"], ref["dL_dsh"], "sh"); close(o["dsc"], ref["dL_dscales"], "scales")
    close(o["drot"], ref["dL_drotations"], "rot"); close(o["dop"], ref["dL_dopacity"].reshape(-1), "opacity")
    # per element: within the a-priori budget around the float64 reference on the same fp32 record (oracle/preprocess64.py)
    r = preprocess64.preprocess_backward64(st, np.concatenate([d2, dc, dop[:, None], dcol, dinv[:, None]], 1))
    worst = check_per_element(dict(means3D=o["dm"], cov3D_precomp=o["dcov"], shs=o["dsh"], scales=o["dsc"], rotations=o["drot"],
                                   opacities=o["dop"]), r, st.radii > 0)
    print("worst |shim - ref64| / budget: " + ", ".join(f"{k} {w:.3g}" for k, w in worst.items()))
    assert all(w <= 1.0 for w in worst.values()), worst


def test_points_pseudomesh_expansion_matches_reference_golden(shim, golden_dir):
    """gs_points: the product's gms_points_face_fwd (CPU build) against PointsGaussianModel.prepare_scaling_rot / get_scaling."""
    g = np.load(os.path.join(golden_dir, "points_model.npz"))
    tri = np.ascontiguousarray(g["triangles"], np.float32)
    P = tri.shape[0]
    xyz = np.zeros((P, 3), np.float32); sl = np.zeros((P, 2), np.float32); rr = np.zeros((P, 4), np.float32)
    sa = np.zeros((P, 3), np.float32); ra = np.zeros((P, 4), np.float32)
    a = _lib.PointsArgs()
    a.P, a.triangles, a.eps = P, tri.ctypes.data, 1e-8
    a.xyz, a.scaling_log, a.rotation_raw, a.scaling_act, a.rotation_act = [x.ctypes.data for x in (xyz, sl, rr, sa, ra)]
    assert shim.shim_points_expand_forward(C.byref(a)) == 0
    np.testing.assert_array_equal(xyz, tri[:, 0])
    np.testing.assert_allclose(sl, g["_scaling"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(rr, g["_rotation"], atol=2e-6)
    np.testing.assert_allclose(sa, g["get_scaling"], rtol=1e-5, atol=1e-12)
    np.testing.assert_allclose(ra, g["get_rotation"], atol=2e-6)


def test_points_prepare_vertices_matches_reference_golden(shim, golden_dir):
    """gs_points: the product's gms_points_vertices_fwd (CPU build) against PointsGaussianModel.prepare_vertices
    (games/flat_splatting/scene/points_gaussian_model.py:28-59), with [P,2] and [P,3] log-scale layouts."""
    g = np.load(os.path.join(golden_dir, "points_model.npz"))
    xyz = np.ascontiguousarray(g["pv_xyz"], np.float32); q = np.ascontiguousarray(g["pv_rotation"], np.float32)
    P = xyz.shape[0]
    for cols in (2, 3):
        sl = np.ascontiguousarray(g["pv_scaling"], np.float32)
        if cols == 3:
            sl = np.ascontiguousarray(np.concatenate([np.full((P, 1), -18.0, np.float32), sl], axis=1))
        tri = np.zeros((P, 3, 3), np.float32)
        a = _lib.PointsVerticesArgs()
        a.P, a.xyz, a.scaling_log, a.scaling_cols = P, xyz.ctypes.data, sl.ctypes.data, cols
        a.rotation_raw, a.triangles = q.ctypes.data, tri.ctypes.data
        assert shim.shim_points_prepare_vertices(C.byref(a)) == 0
        np.testing.assert_array_equal(tri[:, 0], xyz)
        np.testing.assert_allclose(tri, g["pv_triangles"], rtol=0, atol=1e-6)

