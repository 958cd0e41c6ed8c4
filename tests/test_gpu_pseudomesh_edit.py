"""-m gpu: the mesh-driven pseudo-mesh (gms_pseudomesh_bind, gms_pseudomesh_repose, gms_bound_points_render_frame).

1. Binding indices are bit-exact against the numpy oracle (pseudomesh_oracle.py): sizes off the CTA / staging tile, F = 1,
   P = 0, duplicated faces (lowest index wins), degenerate faces (never chosen); a mesh of degenerate faces only is refused.
   They also equal the reference's KD-tree indices of the golden fixture.
2. Coefficients are within 1 ulp of the oracle's rounded double solution wherever the frame's condition number is < 1e6.
3. Re-posing on the rest mesh returns the pseudo-mesh; a rigid motion of the mesh moves it rigidly.
4. MeshBoundPointsRenderer.render(vertices=V) is bit-identical to PointsRenderer.render(triangles=repose_pseudomesh(b, V));
   its sync-free render is bit-identical to its synchronising one under every forward option set; it matches the oracle chain.
5. Gaussians on a face collapsed in the driving pose get radius 0, and the image is that of the model without them.
6. evaluate() matches a per-view loop; bad arguments, and a model pose of the wrong size, type or device, are refused."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import pseudomesh_oracle as orc
from gms_b200 import _lib, expansion, io_image, scenes
from gms_b200.metrics import image_metrics
from gms_b200.model import MeshGaussianModel, PointsModel
from gms_b200.render import MeshBoundPointsRenderer, PointsRenderer
from gpu_helpers import assert_image_parity
from helpers import settings_from_camera
from oracle import expansion as oexp
from oracle import raster

pytestmark = pytest.mark.gpu

BG = (0.2, 0.5, 0.9)
W, H = 400, 300
FWD_OPTION_SETS = [{}, {"sort_impl": 1}, {"bin_impl": 1}, {"key16": 0}, {"composite_fwd": 3}, {"tile_order": 0}]


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


def _soup_near(verts, faces, P, seed, spread=0.02):
    """P small pseudo-triangles scattered over the mesh's surface (float32 numpy [P,3,3])."""
    g = np.random.default_rng(seed)
    fi = g.integers(0, faces.shape[0], P)
    b = g.random((P, 3))
    b /= b.sum(1, keepdims=True)
    c = (b[:, :, None] * verts[faces[fi]]).sum(1) + spread * g.standard_normal((P, 3))
    return (c[:, None, :] + 0.01 * g.standard_normal((P, 3, 3))).astype(np.float32)


def _check_binding(tri, verts, faces):
    b = expansion.bind_pseudomesh(torch.tensor(tri).cuda(), torch.tensor(verts).cuda(), torch.tensor(faces).cuda())
    idx, coeffs, nd, _ = orc.bind(tri, verts, faces)
    assert b.n_degenerate == nd
    np.testing.assert_array_equal(b.face.cpu().numpy(), idx)
    got = b.coeffs.cpu().numpy()
    fv = verts[faces[idx]]
    cond = orc.condition_numbers(*orc.frames(fv[:, 0], fv[:, 1], fv[:, 2])[:3]) if len(idx) else np.zeros(0)
    ok = cond < 1e6
    ulps = np.abs(got.view(np.int32).astype(np.int64) - coeffs.view(np.int32).astype(np.int64))[ok]
    assert ulps.size == 0 or ulps.max() <= 1, ulps.max()
    return b, idx


@pytest.mark.parametrize("F_target,P", [(1500, 1037), (700, 128 * 5 + 1), (2100, 3)])
def test_binding_is_bit_exact_against_the_oracle(F_target, P):
    verts, faces = scenes.object_mesh(F_target)
    assert faces.shape[0] % 512 and faces.shape[0] % 128
    _check_binding(_soup_near(verts, faces, P, F_target), verts, faces)


def test_binding_single_face_and_empty_pseudo_mesh():
    verts = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    faces = np.array([[0, 1, 2]], np.int64)
    b, idx = _check_binding(_soup_near(verts, faces, 200, 1, 0.5), verts, faces)
    assert (idx == 0).all()
    b0, _ = _check_binding(np.zeros((0, 3, 3), np.float32), verts, faces)
    assert b0.P == 0 and expansion.repose_pseudomesh(b0, torch.tensor(verts).cuda()).shape == (0, 3, 3)


def test_binding_ties_go_to_the_lowest_face_index():
    verts, faces = scenes.object_mesh(800)
    dup = np.concatenate([faces, faces[::-1]], 0)          # every face twice: same centroid, same distance
    tri = _soup_near(verts, faces, 900, 3)
    _, idx = _check_binding(tri, verts, dup)
    assert (idx < faces.shape[0]).all()


def test_degenerate_faces_are_never_bound():
    verts, faces = scenes.object_mesh(800)
    faces = faces.copy()
    F = faces.shape[0]
    faces[::7, 1] = faces[::7, 0]                          # zero edge
    verts = np.concatenate([verts, np.array([[0.0, 0.0, 0.0], [0.1, 0.0, 0.0], [0.2, 0.0, 0.0]], np.float32)], 0)
    faces[3::7] = [verts.shape[0] - 3, verts.shape[0] - 2, verts.shape[0] - 1]     # collinear: zero area
    tri = _soup_near(verts, faces, 1200, 4)
    b, idx = _check_binding(tri, verts, faces)
    deg = np.zeros(F, bool)
    deg[::7] = deg[3::7] = True
    assert b.n_degenerate == deg.sum() and not deg[idx].any()


def test_all_degenerate_faces_are_refused():
    verts = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0]], np.float32)
    faces = np.array([[0, 1, 2], [0, 0, 1]], np.int64)
    tri = torch.tensor(_soup_near(verts, np.array([[0, 1, 2]]), 10, 5)).cuda()
    with pytest.raises(ValueError, match="degenerate"):
        expansion.bind_pseudomesh(tri, torch.tensor(verts).cuda(), torch.tensor(faces).cuda())
    a, nd = _bind_args(tri, torch.tensor(verts).cuda(), torch.tensor(faces).cuda())
    assert _lib.lib().gms_pseudomesh_bind(C.byref(a[0]), None) == _lib.GMS_E_ARG and nd.value == 2


def _bind_args(tri, v, f):
    P, F = tri.shape[0], f.shape[0]
    keep = [torch.empty(P, dtype=torch.int32, device="cuda"), torch.empty(P, 3, 3, device="cuda"),
            torch.empty(int(_lib.lib().gms_pseudomesh_bind_scratch_bytes(F)), dtype=torch.uint8, device="cuda")]
    nd = C.c_int32(-1)
    a = _lib.PseudomeshBindArgs()
    a.P, a.triangles, a.V, a.F, a.vertices, a.faces = P, tri.data_ptr(), v.shape[0], F, v.data_ptr(), f.data_ptr()
    a.face, a.coeffs, a.n_degenerate = keep[0].data_ptr(), keep[1].data_ptr(), C.pointer(nd)
    a.scratch, a.scratch_bytes = keep[2].data_ptr(), keep[2].numel()
    return (a, keep), nd


def test_binding_matches_the_reference_kd_tree(golden_dir):
    g = np.load(f"{golden_dir}/pseudomesh_edit.npz")
    b, _ = _check_binding(g["triangles"], g["vertices"], g["faces"])
    np.testing.assert_array_equal(b.face.cpu().numpy(), g["index_of_closest"])
    edited = expansion.repose_pseudomesh(b, torch.tensor(g["vertices_edited"]).cuda()).cpu().numpy()
    idx, coeffs, _, _ = orc.bind(g["triangles"], g["vertices"], g["faces"])
    np.testing.assert_array_equal(edited, orc.repose(idx, coeffs, g["vertices_edited"], g["faces"]))
    err = np.abs(edited - g["edited_triangles"]).max()
    print(f"[pseudomesh edit] max |native - reference edited_triangles| {err:.3g}")
    assert err <= 1e-4


def test_repose_rest_and_rigid_motion():
    verts, faces = scenes.object_mesh(1500)
    tri = _soup_near(verts, faces, 3000, 6)
    b, _ = _check_binding(tri, verts, faces)
    v = torch.tensor(verts).cuda()
    back = expansion.repose_pseudomesh(b, v)
    # |w - v1| <= ~0.1 here: the re-pose rounds a few ops of magnitude <= |v1| + 3 |c|, so a handful of fp32 ulps of ~1.5
    err = float((back - torch.tensor(tri).cuda()).abs().max())
    print(f"[pseudomesh edit] rest-pose round trip max error {err:.3g}")
    assert err <= 2e-6
    ang = 0.7
    R = torch.tensor([[math.cos(ang), -math.sin(ang), 0], [math.sin(ang), math.cos(ang), 0], [0, 0, 1]], dtype=torch.float64)
    R = R @ torch.tensor([[1, 0, 0], [0, math.cos(0.3), -math.sin(0.3)], [0, math.sin(0.3), math.cos(0.3)]], dtype=torch.float64)
    tvec = torch.tensor([0.3, -0.2, 0.5], dtype=torch.float64)
    moved = expansion.repose_pseudomesh(b, (v.double() @ R.T.cuda() + tvec.cuda()).float())
    want = torch.tensor(tri).double() @ R.T + tvec
    err = float((moved.double().cpu() - want).abs().max())
    print(f"[pseudomesh edit] rigid motion max error {err:.3g}")
    assert err <= 4e-6


# ---- rendering
_cache = {}


def _bound_model(degree=3):
    """The pseudo-mesh of a mesh-Gaussian expansion on object_mesh(2000), bound to that mesh."""
    if "m" not in _cache:
        verts, faces = scenes.object_mesh(2000)
        p = scenes.init_mesh_gaussians(verts, faces, K=3, seed=8, trained_like=True)
        with torch.no_grad():
            xyz, sl, rr = MeshGaussianModel.from_params(p, "cuda").expand_fused(activated=False)
        _cache["m"] = (PointsModel.from_gaussians(xyz, sl, rr, p._features_dc, p._features_rest, p._opacity, "cuda"),
                       torch.tensor(verts).cuda(), torch.tensor(faces).cuda())
    pm, v, f = _cache["m"]
    pm.active_sh_degree = degree
    return pm, pm.bind_to_mesh(v, f)


def _camera():
    return scenes.look_at_camera((2.2, 0.7, 1.0), (0, 0, 0), W, H)


def _pose(v, t):
    return scenes.transform_hotdog_fly(v, t)


@pytest.mark.parametrize("t", [None, 0.0, 3.0, 9.0])
def test_bound_render_is_bit_identical_to_the_triangles_render(t):
    pm, bm = _bound_model()
    cam_d, bg = _camera().to("cuda"), torch.tensor(BG, device="cuda")
    V = None if t is None else _pose(bm.vertices, t)
    tri = expansion.repose_pseudomesh(bm.binding, bm.vertices if V is None else V)
    br, pr = MeshBoundPointsRenderer(bm, W, H), PointsRenderer(pm, W, H)
    for _ in range(2):                                   # synchronising, then sync-free
        a = [x.clone() for x in br.render(cam_d, bg, vertices=V)]
        b = [x.clone() for x in pr.render(cam_d, bg, triangles=tri)]
        torch.cuda.synchronize()
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    assert br.overflows == 0 and br.last_num_rendered > 0


@pytest.mark.parametrize("opts", FWD_OPTION_SETS, ids=_opt_id)
def test_sync_free_render_is_bit_identical_to_the_synchronising_one(opts):
    _, bm = _bound_model()
    cam_d, bg = _camera().to("cuda"), torch.tensor(BG, device="cuda")
    V = _pose(bm.vertices, 4.0)
    with _Options(opts):
        r = MeshBoundPointsRenderer(bm, W, H)
        sync = [x.clone() for x in r.render(cam_d, bg, vertices=V)]
        free = [x.clone() for x in r.render(cam_d, bg, vertices=V)]
        torch.cuda.synchronize()
        N = r.last_num_rendered
    assert r.overflows == 0 and r.capacity > N > 0
    for a, b in zip(sync, free):
        assert torch.equal(a, b)


def test_bound_render_matches_the_oracle_chain():
    pm, bm = _bound_model(3)
    cam = _camera()
    cam_d, bg = cam.to("cuda"), torch.tensor(BG, device="cuda")
    V = _pose(bm.vertices, 6.0)
    r = MeshBoundPointsRenderer(bm, W, H)
    r.render(cam_d, bg, vertices=V)
    image, radii, invd = r.render(cam_d, bg, vertices=V)
    tri = expansion.repose_pseudomesh(bm.binding, V)
    xyz, sc, rot = (x.cpu() for x in expansion.points_prepare_scaling_rot(tri, pm.eps_s0, activated=True))
    osl, orr = oexp.points_prepare_scaling_rot(tri.cpu(), pm.eps_s0)
    osc, orot = oexp.points_get_scaling(osl, pm.eps_s0), torch.nn.functional.normalize(orr)
    assert bool(((sc - osc).abs() <= 1e-4 * osc + 1e-7).all()) and float((rot - orot).abs().max()) <= 1e-5
    S = settings_from_camera(cam, sh_degree=3, bg=BG)
    st = raster.forward(S, xyz, torch.sigmoid(pm._opacity.cpu()), shs=pm._features.cpu().contiguous(), scales=sc, rotations=rot)
    np.testing.assert_array_equal(radii.cpu().numpy(), st.radii)
    ok = assert_image_parity(st, image.cpu().numpy())
    assert np.abs(invd.cpu().numpy() - st.invdepth)[:, ok].max() <= 1e-5


def test_gaussians_on_a_collapsed_face_are_not_drawn():
    pm, bm = _bound_model()
    cam_d, bg = _camera().to("cuda"), torch.tensor(BG, device="cuda")
    faces = bm.faces
    face = bm.binding.face.long()
    V = bm.vertices.clone()
    target = faces[face[0]]
    V[target[1]] = V[target[0]]                         # face[0]'s first edge has length 0 -> degenerate in this pose
    tri = expansion.repose_pseudomesh(bm.binding, V)
    bad = ~torch.isfinite(tri).reshape(tri.shape[0], -1).all(1)
    assert bool(bad[face == face[0]].all()) and int(bad.sum()) >= 1
    r = MeshBoundPointsRenderer(bm, W, H)
    r.render(cam_d, bg, vertices=V)
    image, radii, invd = (x.clone() for x in r.render(cam_d, bg, vertices=V))
    torch.cuda.synchronize()
    assert int(radii[bad].abs().max()) == 0 and r.overflows == 0
    keep = ~bad
    kept = PointsModel(tri[keep], pm._features[keep], pm._opacity[keep], pm.active_sh_degree)
    kr = PointsRenderer(kept, W, H)
    want = [x.clone() for x in kr.render(cam_d, bg)]
    assert r.last_num_rendered == kr.last_num_rendered
    assert torch.equal(image, want[0]) and torch.equal(invd, want[2]) and torch.equal(radii[keep], want[1])


@pytest.mark.parametrize("protocol", ["training_report", "metrics"])
def test_evaluate_matches_a_per_view_loop(protocol):
    cams = [c.to("cuda") for c in scenes.ring_cameras(5, 2.6, W, H)]
    g = torch.Generator().manual_seed(5)
    gts = [io_image.to_device_float((torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).cuda()).clone() for _ in cams]
    bg = torch.tensor(BG, device="cuda")
    _, bm = _bound_model()
    bm.vertices = _pose(bm.vertices, 2.0)
    try:
        res = MeshBoundPointsRenderer(bm, W, H).evaluate(cams, gts, bg, protocol=protocol)
        loop = MeshBoundPointsRenderer(bm, W, H)
        for v, (cam, gt) in enumerate(zip(cams, gts)):
            want = image_metrics(loop.render(cam, bg)[0], gt, protocol).cpu()
            assert torch.equal(res.per_view[v].view(torch.int64), want.view(torch.int64)), v
    finally:
        _cache.clear()


def test_render_leaves_the_model_untouched_and_bad_arguments_are_refused():
    pm, bm = _bound_model()
    before = [t.clone() for t in (bm.vertices, bm.binding.face, bm.binding.coeffs, pm._features, pm._opacity)]
    cam_d, bg = _camera().to("cuda"), torch.tensor(BG, device="cuda")
    r = MeshBoundPointsRenderer(bm, W, H)
    r.render(cam_d, bg, vertices=_pose(bm.vertices, 5.0))
    torch.cuda.synchronize()
    for a, b in zip(before, (bm.vertices, bm.binding.face, bm.binding.coeffs, pm._features, pm._opacity)):
        assert torch.equal(a, b)
    with pytest.raises(ValueError):
        r.render(cam_d, bg, vertices=bm.vertices[:-1])
    P = bm.binding.P

    def call(**kw):
        a = _lib.BoundPointsRenderArgs()
        a.P, a.M, a.eps = P, pm._features.shape[1], pm.eps_s0
        a.face, a.coeffs, a.V, a.F = bm.binding.face.data_ptr(), bm.binding.coeffs.data_ptr(), bm.binding.V, bm.faces.shape[0]
        a.vertices, a.faces = bm.vertices.data_ptr(), bm.faces.data_ptr()
        a.features, a.opacity_raw = pm._features.data_ptr(), pm._opacity.data_ptr()
        a.settings.image_width, a.settings.image_height = W, H
        a.settings.viewmatrix = cam_d.world_view_transform.data_ptr()
        a.image, a.invdepth, a.radii = r.image.data_ptr(), r.invdepth.data_ptr(), r.radii.data_ptr()
        a.workspace, a.workspace_bytes = r.ws.data_ptr(), r.ws.numel()
        for k, v in kw.items():
            setattr(a, k, v)
        return _lib.lib().gms_bound_points_render_frame(C.byref(a), r._cb, None, None)

    v, f = bm.vertices, bm.faces
    tri = expansion.repose_pseudomesh(bm.binding, v)
    torch.cuda.synchronize()
    _lib.launch_count(reset=True)
    for kw in ({"face": None}, {"coeffs": None}, {"vertices": None}, {"faces": None}, {"features": None}, {"opacity_raw": None},
               {"image": None}, {"invdepth": None}, {"radii": None}, {"workspace": None}, {"workspace_bytes": r.ws.numel() - 1},
               {"P": -1}, {"F": 0}, {"V": 0}):
        assert call(**kw) == _lib.GMS_E_ARG, kw
        assert b"gms_bound_points_render_frame" in _lib.lib().gms_last_error(), kw
    (a, keep), _ = _bind_args(tri, v, f)
    for k, val in (("P", -1), ("F", 0), ("face", None), ("scratch", None), ("scratch_bytes", keep[2].numel() - 1)):
        old = getattr(a, k)
        setattr(a, k, val)
        assert _lib.lib().gms_pseudomesh_bind(C.byref(a), None) == _lib.GMS_E_ARG, k
        setattr(a, k, old)
    ra = _lib.PseudomeshReposeArgs()
    ra.P, ra.face, ra.coeffs, ra.V, ra.F, ra.vertices, ra.faces, ra.triangles = P, None, None, v.shape[0], f.shape[0], 0, 0, 0
    assert _lib.lib().gms_pseudomesh_repose(C.byref(ra), None) == _lib.GMS_E_ARG
    assert _lib.launch_count(reset=True) == 0
    with pytest.raises(ValueError):
        expansion.bind_pseudomesh(tri, v, f + 1000)
    with pytest.raises(ValueError):
        expansion.bind_pseudomesh(tri[:, :2], v, f)
    with pytest.raises(ValueError):
        expansion.bind_pseudomesh(tri, v, f[:, :2])
    nan_tri = tri.clone()
    nan_tri[0, 0, 0] = float("nan")
    with pytest.raises(ValueError):
        expansion.bind_pseudomesh(nan_tri, v, f)


def test_a_bad_model_pose_is_refused_before_any_launch():
    """The model's pose reaches the kernel as a raw float32 [V,3] device pointer: assigning a pose of the wrong size or on
    the host raises, a float64 pose is stored as float32, and a pose that bypasses the setter is refused by render() and
    evaluate() before anything is launched."""
    _, bm = _bound_model()
    cam_d, bg = _camera().to("cuda"), torch.tensor(BG, device="cuda")
    rest = bm.vertices
    V = _pose(rest, 3.0)
    try:
        r = MeshBoundPointsRenderer(bm, W, H)
        for bad in (V[:-1], torch.cat([V, V[:1]]), V.cpu(), V[:, :2]):
            with pytest.raises(ValueError):
                bm.vertices = bad
            assert bm.vertices is rest
        bm.vertices = V
        want = [x.clone() for x in r.render(cam_d, bg)]
        bm.vertices = V.double()
        assert bm.vertices.dtype == torch.float32 and bm.vertices.is_contiguous()
        got = [x.clone() for x in r.render(cam_d, bg)]
        torch.cuda.synchronize()
        for a, b in zip(want, got):
            assert torch.equal(a, b)
        gt = torch.rand(3, H, W, device="cuda")
        for bad in (V.double(), V[:-1].contiguous(), V.cpu(), V.t().contiguous().t()):
            bm._vertices = bad
            torch.cuda.synchronize()
            _lib.launch_count(reset=True)
            with pytest.raises(RuntimeError, match="pose"):
                r.render(cam_d, bg)
            with pytest.raises(RuntimeError, match="pose"):
                r.evaluate([cam_d], [gt], bg)
            assert _lib.launch_count(reset=True) == 0
    finally:
        bm.vertices = rest
