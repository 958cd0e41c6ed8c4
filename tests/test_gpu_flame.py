"""-m gpu: gs_flame on the library's kernels.

Expansion: the softmax weights on every mesh of tests/expansion_cases.py at K = 1, 3, 7 (per-thread kernels) and K = 40,
100, 128 (warp-per-face kernels), per element against float64 (tests/softmax_expansion_cases.py).
Training: FlameGaussianModel + NativeFrame / FlameTrainer against the reference's op sequence (tests/flame_reference.AtenFlameArm)
on the synthetic FLAME driver (tests/flame_driver.py): loss and gradients of the first step, three steps, launches per step."""
import ctypes as C

import numpy as np
import pytest
import torch

import expansion_cases as ec
import flame_driver
import flame_reference as fr
import softmax_expansion_cases as sc
from gms_b200 import _lib, scenes
from gms_b200.model import FlameGaussianModel
from gms_b200.trainer import FlameTrainer, NativeFrame

pytestmark = pytest.mark.gpu

CASES = sc.build_cases()
# expansion_cases.TOL, but for the vertex gradient of the sliver mesh, which sums the K splats of every face around a vertex:
# its worst normalised error on an H100 (NVIDIA H100 80GB HBM3, 700 W) is 134 at K = 40 (114 at K = 7; relu weights, K = 3: 33)
# The vertex gradient sums, over the faces around a vertex, K splats each; on the sliver mesh (s2 = a2.v2 / 2 cancels) every
# splat's term carries that cancellation, so the error grows with K while the fp32 oracle's per-face error does not.
TOL_SLIVER = dict(ec.TOL, dL_dvertices=320.0)


def _tol(case):
    return TOL_SLIVER if case.name.startswith("sliver") else ec.TOL


def _run(case):
    stream = torch.cuda.current_stream().cuda_stream

    def put(arr):
        t = torch.from_numpy(arr).cuda()
        return t, t.data_ptr()

    def call(fn, *args):
        args[0].alpha_activation = _lib.ALPHA_SOFTMAX
        _lib.check(fn(*[C.byref(x) for x in args], stream), fn.__name__)

    L = _lib.lib()
    return ec.run_abi(case, put, lambda t: t.cpu().numpy(), lambda a: call(L.gms_expand_forward, a),
                      lambda a, g: call(L.gms_expand_backward, a, g))


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_softmax_expansion_kernels_vs_float64(case):
    ec.check_case(sc.Reference(case), _run(case), _tol(case), f"gpu softmax {case.name}")


def test_softmax_expansion_vs_reference_golden():
    """The kernels against tests/golden/flame, written by the reference's own GaussianFlameModel: update_alpha +
    prepare_scaling_rot and the gradients of _alpha, _scales, the driver's raw vertices and _vertices_enlargement."""
    import os
    from gms_b200 import expansion
    from gms_b200.model import flame_transform_vertices
    e = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flame", "expected.npz")))
    cu = lambda k, g=True: torch.tensor(e[k], device="cuda").requires_grad_(g)
    raw, enl, al, sc = cu("raw_vertices"), cu("_vertices_enlargement"), cu("_alpha"), cu("_scales")
    faces = torch.tensor(e["faces"], device="cuda")
    verts = flame_transform_vertices(raw[None], enl)
    xyz, sl, rr, alpha, _ = expansion.expand(verts, faces, al, sc, activated=False, alpha_activation=_lib.ALPHA_SOFTMAX)
    torch.cuda.synchronize()
    for k, t in (("vertices", verts), ("alpha", alpha), ("_xyz", xyz), ("_scaling", sl), ("_rotation", rr)):
        r = e[k]
        err = float(np.abs(t.detach().cpu().numpy() - r).max() / np.abs(r).max())
        assert err <= 2e-6, (k, err)
    g = torch.autograd.grad((xyz * cu("up_xyz", False)).sum() + (sl * cu("up_scaling", False)).sum() +
                            (rr * cu("up_rotation", False)).sum(), (al, sc, raw, enl))
    for k, t in zip(("d_alpha", "d_scales", "d_raw_vertices", "d_vertices_enlargement"), g):
        r = e[k]
        err = float(np.abs(t.cpu().numpy() - r).max() / np.abs(r).max())
        print(f"[flame] golden {k}: max|kernel - reference| / max|reference| {err:.2e}")
        assert err <= 1e-4, (k, err)


def test_bad_alpha_activation_is_refused():
    case = CASES[0]
    a = _lib.ExpandArgs()
    v, f = torch.from_numpy(case.vertices).cuda(), torch.from_numpy(case.faces).cuda()
    al, s = torch.from_numpy(case.alpha_raw).cuda(), torch.from_numpy(case.scale_raw).cuda()
    a.V, a.F, a.K, a.eps = v.shape[0], case.F, case.K, 1e-8
    a.vertices, a.faces, a.alpha_raw, a.scale_raw = v.data_ptr(), f.data_ptr(), al.data_ptr(), s.data_ptr()
    a.alpha_activation = 2
    assert _lib.lib().gms_expand_forward(C.byref(a), torch.cuda.current_stream().cuda_stream) == _lib.GMS_E_ARG


# ---------------------------------------------------------------------------------------------------------- training

def _scene(K=10, rings=23, segments=24, W=256, H=256):
    torch.manual_seed(0)
    drv = flame_driver.SyntheticFlame(rings=rings, segments=segments).cuda()
    faces = torch.from_numpy(drv.faces).cuda()
    m = FlameGaussianModel.create(drv, faces, K=K, seed=3)
    m.active_sh_degree = 1
    cams = [scenes.look_at_camera((0.35 * np.cos(a), 0.1, 0.35 * np.sin(a)), (0, 0, 0), W, H) for a in np.linspace(0, 2 * np.pi, 4, endpoint=False)]
    cams = [c.to("cuda") for c in cams]
    g = torch.Generator(device="cuda").manual_seed(1)
    gts = [torch.rand(3, H, W, device="cuda", generator=g) for _ in cams]
    return m, cams, gts, torch.tensor([1.0, 1.0, 1.0], device="cuda")


@pytest.mark.parametrize("K", [10, 100])
def test_first_step_loss_and_gradients_match_the_reference_arm(K):
    """K = 100 runs the warp-per-face kernels inside gms_train_frame (softmax weights, K >= 16); K = 10 the per-thread ones."""
    m, cams, gts, bg = _scene(K=K)
    arm = fr.AtenFlameArm(m, bg)
    t = FlameTrainer(m, bg)
    # the native frame's gradients, before any optimizer step
    verts = m.driver_vertices()
    with torch.no_grad():
        m.vertices.copy_(verts)
    m.vertices.grad.zero_()
    frame = NativeFrame(m, cams[0].image_width, cams[0].image_height, sync_free=False)
    names = fr.AtenFlameArm.NAMES + ("_alpha", "_scales", "_opacity")
    frame.run(cams[0], gts[0], bg)          # a first run: the native gradients' run-to-run noise (float atomics)
    torch.autograd.backward(verts, m.vertices.grad, retain_graph=True)
    first = {n: getattr(m, n).grad.clone() for n in names}
    t.adam.zero_grad()
    m.vertices.grad.zero_()
    loss = float(frame.run(cams[0], gts[0], bg))
    torch.autograd.backward(verts, m.vertices.grad)
    ref = float(arm.step(cams[0], gts[0], optimizer_step=False))
    print(f"[flame] first-step loss native {loss:.9f} reference {ref:.9f}")
    assert abs(loss - ref) <= 1e-6 * max(1.0, abs(ref))
    # The arm's fp32 ATen expansion rounds differently from the kernels, so the two differ by more than the native frame's
    # run-to-run noise (printed): a fixed level, 2.5-3.5x the worst measured on an H100 (NVIDIA H100 80GB HBM3, 700 W):
    # 2.8e-4 of max|reference| at K = 10, 4.2e-3 (opacity) at K = 100, where a 1e5-Gaussian image moves more pixels.
    level = 1e-3 if K <= 10 else 1.5e-2
    for n in names:
        g, r = getattr(m, n).grad, arm.p[n].grad
        d, noise, top = float((g - r).abs().max()), float((g - first[n]).abs().max()), float(r.abs().max())
        print(f"[flame] K={K} first-step gradient {n}: max|native - reference| / max|reference| {d / top:.2e}, run-to-run {noise / top:.2e}")
        assert d <= level * top, n
    t.adam.zero_grad()


def _three_steps(K, arm=False):
    m, cams, gts, bg = _scene(K=K)
    a = fr.AtenFlameArm(m, bg) if arm else None
    t = FlameTrainer(m, bg)
    launches, losses = [], []
    for i in range(3):
        _lib.launch_count(reset=True)
        ln = float(t.step(cams[i % 4], gts[i % 4]))
        torch.cuda.synchronize()
        launches.append(_lib.launch_count())
        losses.append((ln, float(a.step(cams[i % 4], gts[i % 4])) if arm else None))
    return m, a, launches, losses


@pytest.mark.parametrize("K", [10, 100])
def test_trainer_tracks_the_reference_arm_and_launch_count(K):
    """Three steps against the reference arm.  The bound on each parameter is the run-to-run noise method of DESIGN.md 4.2:
    10x the largest difference between two native runs from the same start (float atomics in the composite and vertex
    backward), or 1 % of the group's learning rate if that is larger (a level 100x under what one Adam step moves).
    Adam (eps 1e-15) moves an element whose gradient is at the level of that noise by about +/- lr whatever its size, so
    on the K = 100 model a few such elements (of 1e5 opacities and scales) may take opposite steps in the two arms: at most
    max(2, 1e-4 of the elements) may exceed the bound, and none may exceed what three Adam steps can move (6 lr)."""
    m, arm, launches, losses = _three_steps(K, arm=True)
    m2, _, _, _ = _three_steps(K)
    print(f"[flame] K={K} losses (native, reference) {losses}; library launches per step {launches}")
    for ln, lr in losses:
        assert abs(ln - lr) <= 1e-4 * abs(lr)
    assert launches[1:] == [13, 13]
    for n in fr.AtenFlameArm.NAMES + ("_alpha", "_scales", "_opacity"):
        p, r, p2 = getattr(m, n).detach(), arm.p[n].detach(), getattr(m2, n).detach()
        lr = next(g["lr"] for g in arm.adam.param_groups if g["name"] == n)
        d, noise = float((p - r).abs().max()), float((p - p2).abs().max())
        bound = max(10 * noise, 1e-2 * lr)
        over = int(((p - r).abs() > bound).sum())
        print(f"[flame] K={K} after 3 steps {n}: max|native - reference| {d:.3e}, native run-to-run {noise:.3e}, bound {bound:.3e}, "
              f"{over} of {p.numel()} over it")
        assert over <= max(2, 1e-4 * p.numel()) and d <= 6 * lr, n


def test_softmax_segments_render():
    """A segmented model (K = 3 and K = 100 meshes, one expansion launch each) with softmax weights through gms_render_frame,
    against the per-mesh softmax expansion concatenated and drawn by the shim rasterizer."""
    import diff_gaussian_rasterization as dgr
    from gms_b200 import expansion
    from gms_b200.model import MultiMeshGaussianModel
    from gms_b200.render import NativeRenderer
    plist = []
    for k, (K, lvl) in enumerate(((3, 2), (100, 1))):
        v, f = scenes.icosphere(lvl, radius=0.35 + 0.05 * k)
        p = scenes.init_mesh_gaussians(v + np.float32([0.8 * k - 0.4, 0.1 * k, 0]), f, K=K, seed=5 + k, trained_like=True)
        p._alpha = 2.0 * torch.randn(p._alpha.shape, generator=torch.Generator().manual_seed(9 + k))
        plist.append(p)
    m = MultiMeshGaussianModel.from_mesh_params(plist, "cuda", packed_features=True, segmented=True)
    m.alpha_activation = _lib.ALPHA_SOFTMAX
    W, H = 256, 256
    cam = scenes.look_at_camera((0.4, 1.2, 2.6), (0.0, 0.0, 0.0), W, H).to("cuda")
    bg = torch.tensor([1.0, 1.0, 1.0], device="cuda")
    r = NativeRenderer(m, W, H)
    img, radii = (t.clone() for t in r.render(cam, bg)[:2])          # synchronising
    img2, radii2 = (t.clone() for t in r.render(cam, bg)[:2])        # sync-free
    assert torch.equal(img, img2) and torch.equal(radii, radii2)
    outs = [expansion.expand(m.vertices.detach(), f, a.detach(), s.detach(), alpha_activation=_lib.ALPHA_SOFTMAX)[:3]
            for f, a, s in m.mesh_views()]
    xyz, sc, rot = (torch.cat([o[i] for o in outs]) for i in range(3))
    rs = dgr.GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=bg,
                                           scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
                                           sh_degree=m.active_sh_degree, campos=cam.camera_center, prefiltered=False, debug=False,
                                           antialiasing=False)
    with torch.no_grad():
        ref, rradii, _ = dgr.GaussianRasterizer(raster_settings=rs)(means3D=xyz, means2D=torch.zeros_like(xyz), opacities=m.get_opacity,
                                                                     shs=m.get_features, scales=sc, rotations=rot)
    d = float((img - ref).abs().max())
    print(f"[flame] segmented softmax render vs per-mesh expansion + shim: max |diff| {d:.2e}, radii differ {int((radii != rradii).sum())}")
    assert torch.equal(radii, rradii) and d <= 1e-5


def test_native_renderer_draws_the_flame_model():
    """NativeRenderer on a FlameGaussianModel: the current pose with softmax weights, as training_report renders it."""
    from gms_b200.render import NativeRenderer
    m, cams, gts, bg = _scene()
    arm = fr.AtenFlameArm(m, bg)
    r = NativeRenderer(m, cams[0].image_width, cams[0].image_height)
    for cam in cams:
        img = r.render(cam, bg)[0].clone()
        with torch.no_grad():
            ref = arm.render(cam)
        d, mean = float((img - ref).abs().max()), float((img - ref).abs().mean())
        print(f"[flame] native render vs reference arm: max |diff| {d:.2e}, mean {mean:.2e}")
        # the two expansions differ in the last bits (fp32 ATen against the kernel); a Gaussian at a culling or tile threshold
        # then moves a few pixels (5.5e-4 measured on an H100)
        assert mean <= 1e-6 and d <= 5e-3


def test_flame_renderer_matches_free_renderer_and_animates():
    """FlameRenderer (gms_flame_render_frame) on a checkpoint written by io_ply.save_flame_model: at the trained pose it draws
    what NativeFreeRenderer draws of the same point_cloud.ply as a gs model (README: renders_gs_flame == renders_gs); an
    --animated expression moves it; sync-free renders equal the synchronising one bit for bit."""
    import tempfile
    from gms_b200 import io_ply
    from gms_b200.model import FlameCheckpoint, FreeGaussianModel
    from gms_b200.render import FlameRenderer, NativeFreeRenderer
    m, cams, gts, bg = _scene(K=100)
    t = FlameTrainer(m, bg)
    for i in range(2):
        t.step(cams[i], gts[i])
    with tempfile.TemporaryDirectory() as d:
        ply = f"{d}/point_cloud.ply"
        io_ply.save_flame_model(ply, m)
        ck = FlameCheckpoint.load(ply, active_sh_degree=m.active_sh_degree)
        free = FreeGaussianModel.from_checkpoint(ply, kind="gs", device="cuda", active_sh_degree=m.active_sh_degree)
    ck.vertices = ck.driver_vertices(m.driver)
    W, H = cams[0].image_width, cams[0].image_height
    r, rf = FlameRenderer(ck, W, H), NativeFreeRenderer(free, W, H)
    for cam in cams:
        img, radii = (x.clone() for x in r.render(cam, bg)[:2])
        img_s, radii_s = (x.clone() for x in r.render(cam, bg)[:2])
        assert torch.equal(img, img_s) and torch.equal(radii, radii_s)
        fimg, fradii = (x.clone() for x in rf.render(cam, bg)[:2])
        diff = (radii != fradii).sum().item()
        dimg = float((img - fimg).abs().max())
        print(f"[flame] FlameRenderer vs NativeFreeRenderer: max |diff| {dimg:.2e}, radii differ {diff} of {radii.numel()}")
        assert diff <= 1e-3 * radii.numel() and dimg <= 1e-3
    exp = ck._flame_exp.clone()
    exp[0, [0, 5, 7, 9]] = 2.0
    va = ck.driver_vertices(m.driver, expression_params=exp)
    assert float((va - ck.vertices).abs().max()) > 1e-4
    img_a = r.render(cams[0], bg, vertices=va)[0].clone()
    # the animated frame against the same protocol in ATen: xyz = alpha @ vertices[faces], checkpoint scales / rotations
    import diff_gaussian_rasterization as dgr
    xyz = torch.matmul(ck.alpha, va[ck.faces]).reshape(-1, 3)
    cam = cams[0]
    rs = dgr.GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=bg,
                                           scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
                                           sh_degree=ck.active_sh_degree, campos=cam.camera_center, prefiltered=False, debug=False,
                                           antialiasing=False)
    with torch.no_grad():
        ref = dgr.GaussianRasterizer(raster_settings=rs)(means3D=xyz, means2D=torch.zeros_like(xyz), opacities=torch.sigmoid(ck._opacity),
                                                         shs=ck._features, scales=torch.exp(ck._scaling),
                                                         rotations=torch.nn.functional.normalize(ck._rotation))[0]
    da = float((img_a - ref).abs().max())
    print(f"[flame] animated FlameRenderer vs ATen protocol: max |diff| {da:.2e}")
    assert da <= 1e-3
