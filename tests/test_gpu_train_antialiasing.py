"""-m gpu: training with antialiasing (the reference's pipe.antialiasing) on the one-call frames, for gs_mesh, segmented
gs_multi_mesh, gs_flame, gs and gs_flat.

With the flag on, the preprocess forward scales each splat's opacity by h = sqrt(max(2.5e-5, det_cov / det_cov_dilated)) and
the backward carries dL/dh into the 2D covariance.  Checked here: an antialiased training frame against the same step
through the drop-in rasterizer with antialiasing=True, the ATen expansion / activations and the ATen loss; the fused SH Adam
step with the flag on; the antialiasing term's own gradient on splats either side of the 2.5e-5 floor; the fused
densification statistics; the sync-free loop, a forced capacity overflow and a small view in a larger frame; evaluate()
and resuming; and that the default (antialiasing=False) launches what it launched before."""
import numpy as np
import pytest
import torch

import aten_reference
import diff_gaussian_rasterization as dgr
import mesh_types_cases
import raster_edge_cases as rec
from flame_reference import softmax_expand
from gms_b200 import _lib, dataset, scenes
from gms_b200.flame import NativeFlame
from gms_b200.model import FlameGaussianModel, FreeGaussianModel, MeshGaussianModel, MultiMeshGaussianModel
from gms_b200.render import NativeFreeRenderer, NativeRenderer
from gms_b200.trainer import (FlameOptimizationParams, FlameTrainer, FreeOptimizationParams, FreeTrainer, MeshTrainer,
                              NativeFreeFrame)
from helpers import random_gaussians
from oracle import expansion as oexp
from test_gpu_train_mixed_sizes import _bound, _outputs, _rel

pytestmark = pytest.mark.gpu

# The arm's fp32 ATen expansion and activations round differently from the kernels: on top of the spread bound, the frame
# and the arm may differ by test_gpu_flame's level for that rounding (1e-3 of max |reference| at K = 10).
ARM_LEVEL = 1e-3

TYPES = ["gs_mesh", "gs_multi_mesh", "gs_flame", "gs", "gs_flat"]
MESH_TYPES = ("gs_mesh", "gs_multi_mesh")
FREE_TYPES = ("gs", "gs_flat")
LAMBDA = 0.2
BG = (0.2, 0.5, 0.9)
W, H = 256, 176
NUM_SPLATS = (2, 4, 5)          # gs_multi_mesh: --num_splats 2 4 5, one segment per mesh


def _model(gs_type, degree=3):
    if gs_type == "gs_mesh":
        return MeshGaussianModel.from_params(scenes.init_mesh_gaussians(*scenes.icosphere(3, 0.8), K=3, seed=1), "cuda",
                                             active_sh_degree=degree, packed_features=True)
    if gs_type == "gs_multi_mesh":
        p = []
        for k, (K, lvl, r) in enumerate(zip(NUM_SPLATS, (2, 1, 1), (0.6, 0.35, 0.3))):
            v, f = scenes.icosphere(lvl, r)
            p.append(scenes.init_mesh_gaussians(v + np.float32([0.45 * k - 0.45, 0.1 * k, 0.05 * k]), f, K=K, seed=2 + k))
        m = MultiMeshGaussianModel.from_mesh_params(p, "cuda", active_sh_degree=degree, packed_features=True)
        assert m.segments == [(f.shape[0], K) for f, K in zip((q.faces for q in p), NUM_SPLATS)]
        return m
    if gs_type == "gs_flame":
        init = dataset.flame_init(mesh_types_cases.FLAME_MODEL)
        m = FlameGaussianModel.create(NativeFlame.from_model_file(mesh_types_cases.FLAME_MODEL), init.faces, K=10, seed=4)
        with torch.no_grad():           # non-zero SH rows above the DC term, so degree 3 has something to differentiate
            m._features[:, 1:] = 0.2 * torch.randn(m._features[:, 1:].shape, device="cuda",
                                                   generator=torch.Generator(device="cuda").manual_seed(5))
        m.active_sh_degree = degree
        return m
    g = random_gaussians(3000, seed=5, extent=0.8, flat_frac=0.0)
    s = torch.log(g["scales"])
    return FreeGaussianModel(g["means3D"], (s[:, 1:] if gs_type == "gs_flat" else s).contiguous(), g["rotations"], g["shs"],
                             torch.logit(g["opacities"]), gs_type, "cuda", degree)


def _names(gs_type):
    if gs_type in MESH_TYPES:
        return ("vertices", "_alpha", "_scale", "_features", "_opacity")
    if gs_type == "gs_flame":
        return FlameGaussianModel.FLAME_NAMES + ("_alpha", "_scales", "_features", "_opacity")
    return FreeGaussianModel.NAMES


def _trainer(gs_type, model, antialiasing=True, iterations=1, max_size=None, **free):
    bg = torch.tensor(BG, device="cuda")
    if gs_type in MESH_TYPES:
        return MeshTrainer(model, bg, LAMBDA, native=True, optimizer_step=iterations > 1, max_size=max_size,
                           antialiasing=antialiasing)
    if gs_type == "gs_flame":
        return FlameTrainer(model, bg, FlameOptimizationParams(iterations=iterations), max_size=max_size, antialiasing=antialiasing)
    return FreeTrainer(model, bg, 1.0, FreeOptimizationParams(iterations=iterations, **free), max_size=max_size,
                       antialiasing=antialiasing)


def _frame(tr):
    return tr._frame if isinstance(tr, MeshTrainer) else tr.frame


def _cams(n=4, w=W, h=H):
    cams = []
    for k, c in enumerate(scenes.ring_cameras(n, 2.6, w, h, phase=0.3)):
        c.uid = ("view", k)
        cams.append(c.to("cuda"))
    return cams


def _gts(n=4, w=W, h=H, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(3, h, w, generator=g).cuda() for _ in range(n)]


def _views(gs_type, n=4, w=W, h=H, seed=0):
    return _cams(n, w, h), _gts(n, w, h, seed)


def _step(tr, gs_type, cam, gt):
    """One trainer step whose before_update hook copies the frame's gradients; the frame's outputs after it."""
    grads = {}

    def grab():
        for n in _names(gs_type):
            grads[n] = getattr(tr.model, n).grad.detach().clone()

    tr.step(cam, gt, before_update=grab)
    torch.cuda.synchronize()
    out = _outputs(_frame(tr), cam)
    out["grads"] = grads
    return out


# ---------------------------------------------------------------------------------------------- the autograd arm

def _settings(cam, degree, antialiasing):
    return dgr.GaussianRasterizationSettings(
        image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
        bg=torch.tensor(BG, device="cuda"), scale_modifier=1.0, viewmatrix=cam.world_view_transform,
        projmatrix=cam.full_proj_transform, sh_degree=degree, campos=cam.camera_center, prefiltered=False, debug=False,
        antialiasing=antialiasing)


def aten_arm(gs_type, model, cam, gt, antialiasing=True):
    """The step through autograd, the reference's way: the ATen expansion (oracle/expansion.py, or softmax weights for
    gs_flame) or the ATen activations, the drop-in rasterizer with `antialiasing`, the ATen L1 + SSIM loss.  Leaves are
    copies of the model's tensors (gs_flame: its current vertices; the FLAME tensors' gradients are that vertex gradient
    pulled back through the driver).  -> image, radii, loss, gradients by name, dL/dmeans2D."""
    leaf = lambda t: t.detach().clone().requires_grad_(True)
    m = model
    if gs_type == "gs_flame":
        L = {n: leaf(getattr(m, n)) for n in ("vertices", "_alpha", "_scales", "_features", "_opacity")}
        xyz, sl, rr, _, _ = softmax_expand(L["vertices"], m.faces, L["_alpha"], L["_scales"], m.eps_s0)
        scales = torch.exp(sl)
    elif gs_type in MESH_TYPES:
        L = {n: leaf(getattr(m, n)) for n in _names(gs_type)}
        if m.segments is None:
            xyz, sl, rr, _, _ = oexp.expand(L["vertices"], m.faces, L["_alpha"], L["_scale"], m.eps_s0)
        else:
            views, f0, g0 = [], 0, 0
            for F, K in m.segments:
                views.append((m.faces[f0:f0 + F], L["_alpha"][g0:g0 + F * K].view(F, K, 3), L["_scale"][g0:g0 + F * K]))
                f0, g0 = f0 + F, g0 + F * K
            xyz, sl, rr = oexp.expand_multi([L["vertices"]] * len(views), *zip(*views), eps=m.eps_s0)
        scales = torch.exp(sl)
    else:
        L = {n: leaf(getattr(m, n)) for n in _names(gs_type)}
        xyz, rr, s = L["_xyz"], L["_rotation"], torch.exp(L["_scaling"])
        scales = s if gs_type == "gs" else torch.cat([torch.full((s.shape[0], 1), m.eps_s0, device="cuda"), s], 1)
    m2d = torch.zeros_like(xyz, requires_grad=True)
    image, radii, _ = dgr.GaussianRasterizer(raster_settings=_settings(cam, m.active_sh_degree, antialiasing))(
        means3D=xyz, means2D=m2d, opacities=torch.sigmoid(L["_opacity"]), shs=L["_features"], scales=scales,
        rotations=torch.nn.functional.normalize(rr))
    loss = aten_reference.training_loss(image, gt, LAMBDA)
    loss.backward()
    grads = {n: t.grad for n, t in L.items()}
    if gs_type == "gs_flame":
        flame = [getattr(m, n) for n in FlameGaussianModel.FLAME_NAMES]
        pulled = torch.autograd.grad(m.driver_vertices(), flame, grad_outputs=grads.pop("vertices"))
        grads.update(zip(FlameGaussianModel.FLAME_NAMES, pulled))
    torch.cuda.synchronize()
    return image.detach(), radii, loss.detach(), grads, m2d.grad


def _renderer(gs_type, model, cam):
    cls = NativeFreeRenderer if gs_type in FREE_TYPES else NativeRenderer
    return cls(model, int(cam.image_width), int(cam.image_height))


# ------------------------------------------------------------------------------------- 1. frames against the arm

@pytest.mark.parametrize("degree", [0, 3])
@pytest.mark.parametrize("gs_type", TYPES)
def test_aa_frame_matches_the_autograd_arm(gs_type, degree):
    """One antialiased training frame (the trainer's, sync-free after a first synchronising one) against the autograd arm
    with antialiasing=True: image and radii bit for bit with the native forward renderer drawing the same model with
    antialiasing (pinned to the oracle by test_gpu_render_eval) and the image within 1e-4 of the arm's; the loss to 2e-6
    relative; every raw-parameter gradient within the spread bound of the frame tests (DESIGN.md 4.3) or 10x the frame's
    own run-to-run spread, or ARM_LEVEL for the arm's own rounding.  The arm without antialiasing is further from the frame
    than the arm with it."""
    m = _model(gs_type, degree)
    tr = _trainer(gs_type, m)
    assert tr.antialiasing
    cams, gts = _views(gs_type, 1)
    cam, gt = cams[0], gts[0]
    a1 = _step(tr, gs_type, cam, gt)
    a2 = _step(tr, gs_type, cam, gt)
    assert _frame(tr).capacity > 0 and _frame(tr).overflows == 0
    image, radii, _ = _renderer(gs_type, m, cam).render(cam, torch.tensor(BG, device="cuda"), antialiasing=True)
    torch.cuda.synchronize()
    assert int((a2["radii"] > 0).sum()) > 100, "the view must see the model"
    for x in (a1, a2):
        assert torch.equal(x["image"], image) and torch.equal(x["radii"], radii)
    plain = _renderer(gs_type, m, cam).render(cam, torch.tensor(BG, device="cuda"))[0]
    assert not torch.equal(plain, image), "antialiasing must change the image"
    img, rradii, loss, ref, _ = aten_arm(gs_type, m, cam, gt, antialiasing=True)
    _, _, _, ref_plain, _ = aten_arm(gs_type, m, cam, gt, antialiasing=False)
    d_img = float((img - a2["image"]).abs().max())
    assert d_img <= 1e-4, d_img
    for x in (a1, a2):
        assert abs(float(x["loss"][0]) - float(loss)) <= 2e-6 * abs(float(loss)), (float(x["loss"][0]), float(loss))
    msg = []
    for n in _names(gs_type):
        spread, got = _rel(a1["grads"][n], a2["grads"][n]), _rel(a2["grads"][n], ref[n])
        msg.append(f"{n} {got:.1e} (run-to-run {spread:.1e}, arm without AA {_rel(a2['grads'][n], ref_plain[n]):.1e})")
        assert got <= max(_bound(n), 10 * spread, ARM_LEVEL), (n, got, spread)
    assert _rel(a2["grads"]["_opacity"], ref["_opacity"]) < _rel(a2["grads"]["_opacity"], ref_plain["_opacity"])
    print(f"[{gs_type} D={degree} AA vs autograd arm] image {d_img:.1e}; grad |diff| / max|grad|: " + ", ".join(msg))


@pytest.mark.parametrize("gs_type", ["gs_mesh", "gs_flat"])
def test_aa_fused_sh_adam_equals_unfused_step(gs_type):
    """Antialiased steps with the SH Adam update fused into the frame against the same steps with the frame writing the SH
    gradient and FlatAdam stepping it (a before_update hook turns the fusion off), from the same parameters: 3 steps, the
    SH coefficients within 10x the fused runs' run-to-run spread or 1 % of the learning rate, at most max(2, 1e-4 of the
    elements) over it (Adam moves an element whose gradient is at the float-atomic noise by about +/- lr), none by more than
    6 lr."""
    cams, gts = _views(gs_type, 3)
    runs = []
    for fused in (True, True, False):
        m = _model(gs_type)
        tr = _trainer(gs_type, m, iterations=10)
        for i in range(3):
            tr.step(cams[i], gts[i], before_update=None if fused else (lambda: None))
        torch.cuda.synchronize()
        runs.append(m._features.detach().clone())
    a, a2, b = runs
    lr = 0.0025
    noise = float((a - a2).abs().max())
    bound = max(10 * noise, 1e-2 * lr / 20)
    over = int(((a - b).abs() > bound).sum())
    print(f"[{gs_type} AA fused SH Adam] max|fused - unfused| {float((a - b).abs().max()):.3e}, run-to-run {noise:.3e}, "
          f"{over} of {a.numel()} over {bound:.3e}")
    assert over <= max(2, 1e-4 * a.numel()) and float((a - b).abs().max()) <= 6 * lr


# --------------------------------------------------------------------------- 2. the antialiasing term trains

def _floor_scene():
    """raster_edge_cases.antialiasing's scene (splats 1 % below and 1 % above the 2.5e-5 floor among ordinary ones) as free
    Gaussians.  The tiny splats' zero third scale becomes 1e-6 of their in-plane scale (a log-scale parameter must be
    finite); the oracle's h = opacity' / opacity is read again on these inputs and must still put three splats on the floor
    and three above it."""
    S, g = rec.antialiasing()
    g = dict(g)
    sc = g["scales"].clone()
    sc[:6, 2] = 1e-6 * sc[:6, 0]
    g["scales"] = sc
    st = rec.oracle_forward(S, g)
    h = (st.conic_opacity[:, 3] / g["opacities"][:, 0].numpy()).astype(np.float64)
    floor = float(np.sqrt(np.float32(rec.AA_FLOOR)))
    assert (np.abs(h[:3] - floor) <= 1e-6 * floor).all() and (h[3:6] > floor * (1 + 2e-3)).all(), h[:6]
    return S, g, h, st


def _free_frame_grads(g, logit, cam, gt, antialiasing):
    m = FreeGaussianModel(g["means3D"], torch.log(g["scales"]), g["rotations"], g["shs"], logit, "gs", "cuda", 3)
    from gms_b200.optim import FlatAdam, free_model_groups
    FlatAdam(free_model_groups(m, 1e-3))
    fr = NativeFreeFrame(m, cam.image_width, cam.image_height, LAMBDA, sync_free=False)
    fr.run(cam, gt, torch.tensor(BG, device="cuda"), stats=False, antialiasing=antialiasing)
    torch.cuda.synchronize()
    return {n: getattr(m, n).grad.detach().double().cpu() for n in m.NAMES}, _outputs(fr, cam)


def test_aa_term_trains_either_side_of_the_floor():
    """The antialiased frame against a frame without antialiasing whose opacities are the antialiased ones (sigmoid(logit')
    = y h, h the oracle's): the two draw the same image, so dL/d(y h) is shared and the opacity-logit gradients must differ
    by h y (1 - y) / (y' (1 - y')), the factor the chain rule predicts.  On the floor no gradient flows through
    det_cov / det: the scale gradients of those splats are the non-antialiased frame's; just above it, the term adds a
    gradient of the size of the splat's own."""
    S, g, h, _ = _floor_scene()
    cam = rec.camera(S.image_width, S.image_height).to("cuda")
    gt = torch.rand(3, S.image_height, S.image_width, generator=torch.Generator().manual_seed(9)).cuda()
    y = g["opacities"].double()[:, 0].numpy()
    ye = y * h
    logit = torch.logit(g["opacities"])
    logit_e = torch.tensor(np.log(ye / (1 - ye)), dtype=torch.float32)[:, None]
    ga, oa = _free_frame_grads(g, logit, cam, gt, True)
    gb, ob = _free_frame_grads(g, logit_e, cam, gt, False)
    d_img = float((oa["image"] - ob["image"]).abs().max())
    assert d_img <= 1e-6, d_img
    want = h * y * (1 - y) / (ye * (1 - ye))
    got = ga["_opacity"][:, 0].numpy() / gb["_opacity"][:, 0].numpy()
    ratio_err = np.abs(got[:6] / want[:6] - 1)
    scale_a, scale_b = ga["_scaling"][:6], gb["_scaling"][:6]
    rel = ((scale_a - scale_b).abs().amax(1) / scale_b.abs().amax(1).clamp_min(1e-30)).numpy()
    print(f"[AA floor] h / floor {h[:6] / np.sqrt(rec.AA_FLOOR)}, opacity-logit gradient ratio error {ratio_err}, "
          f"scale gradient |AA - matched| / |matched| {rel}")
    assert (np.abs(gb["_opacity"][:6, 0].numpy()) > 0).all(), "every tiny splat must receive an opacity gradient"
    assert (ratio_err <= 1e-3).all(), ratio_err
    assert (rel[:3] <= 1e-2).all(), rel[:3]
    assert (rel[3:] >= 0.1).all(), rel[3:]


# ---------------------------------------------------------------------------------------------- 3. densification

@pytest.mark.parametrize("gs_type", FREE_TYPES)
def test_aa_densification_statistics_are_the_arm_means2d_norms(gs_type):
    """The fused accum / denom of an antialiased frame: denom is 1 on the frame's visible Gaussians, accum the norm of the
    autograd arm's dL/dmeans2D[:, :2] there, within the xyz spread bound or 10x the frame's run-to-run spread."""
    cams, gts = _views(gs_type, 1)
    stats = []
    for _ in range(2):
        m = _model(gs_type)
        tr = _trainer(gs_type, m)
        out = _step(tr, gs_type, cams[0], gts[0])
        stats.append((tr.frame.accum.clone(), tr.frame.denom.clone(), out["radii"]))
    (acc, den, radii), (acc2, _, _) = stats
    _, _, _, _, m2d = aten_arm(gs_type, m, cams[0], gts[0])
    vis = radii > 0
    assert torch.equal(den, vis.float())
    want = torch.where(vis, torch.norm(m2d[:, :2], dim=-1), torch.zeros_like(acc))
    got, spread = _rel(acc, want), _rel(acc, acc2)
    print(f"[{gs_type} AA statistics] accum |diff| / max {got:.1e}, run-to-run {spread:.1e}")
    assert got <= max(_bound("_xyz"), 10 * spread), (got, spread)


# --------------------------------------------------------------------------------------- 4. sync-free and sizes

@pytest.mark.parametrize("gs_type", TYPES)
def test_aa_loop_is_sync_free_recovers_from_overflow_and_runs_small_views(gs_type):
    """An antialiased loop (Adam on) never synchronises after each view's first frame; a forced overflow renders the
    background and the view's next frame recovers; a small view in a frame sized for a larger one is the exact-size
    antialiased frame, image bit for bit."""
    cams, gts = _views(gs_type, 4)
    m = _model(gs_type)
    tr = _trainer(gs_type, m, iterations=100)
    seen, losses = set(), []
    try:
        for it in range(16):
            v = it % 4
            torch.cuda.set_sync_debug_mode(0 if v not in seen else "error")
            seen.add(v)
            losses.append(tr.step(cams[v], gts[v]).clone())
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert bool(torch.isfinite(torch.stack(losses)).all())
    fr = _frame(tr)
    assert fr.overflows == 0
    fr.capacity_override = max(fr.last_num_rendered // 3, 1)
    tr.step(cams[0], gts[0])
    torch.cuda.synchronize()
    out = _outputs(fr, cams[0])
    assert fr.last_num_rendered > fr.capacity and fr.overflows == 1       # (reading N harvests the frame's slot)
    assert torch.equal(out["image"], torch.tensor(BG, device="cuda")[:, None, None].expand(3, H, W))
    fr.capacity_override = None
    tr.step(cams[0], gts[0])
    torch.cuda.synchronize()
    assert fr.overflows == 1 and fr.capacity >= fr.last_num_rendered > 0
    # a 144 x 112 view: in a frame sized for 256 x 176, and in its own exact-size frame (same model, no Adam step)
    sw, sh = 144, 112
    small = _cams(1, sw, sh)[0]
    sgt = _gts(1, sw, sh, seed=4)[0]
    big = _trainer(gs_type, m, max_size=(W, H))
    exact = _trainer(gs_type, m)
    b = [_step(big, gs_type, small, sgt) for _ in range(2)][-1]
    e = [_step(exact, gs_type, small, sgt) for _ in range(2)][-1]
    assert (_frame(big).W, _frame(big).H) == (W, H) and (_frame(exact).W, _frame(exact).H) == (sw, sh)
    for k in ("radii", "image", "invdepth"):
        assert torch.equal(b[k], e[k]), k


# ------------------------------------------------------------------------------------------ 5. evaluate, resume

@pytest.mark.parametrize("gs_type", TYPES)
def test_aa_evaluate_and_resume(gs_type):
    """evaluate() of an antialiased trainer is NativeRenderer.evaluate(..., antialiasing=True) bit for bit; state_dict ->
    load_state_dict into a fresh antialiased trainer restores every parameter and moment bit for bit and records the flag;
    loading it into a trainer without antialiasing (or a non-antialiased state into an antialiased one) raises, naming
    both settings."""
    cams, gts = _views(gs_type, 4)
    m = _model(gs_type)
    tr = _trainer(gs_type, m, iterations=100)
    for i in range(3):
        tr.step(cams[i], gts[i])
    e = tr.evaluate(cams, gts)
    want = []
    for c, g in zip(cams, gts):
        want.append(_renderer(gs_type, m, c).evaluate([c], [g], torch.tensor(BG, device="cuda"), antialiasing=True).per_view[0])
    assert torch.equal(e.per_view, torch.stack(want))
    plain = _renderer(gs_type, m, cams[0]).evaluate(cams, gts, torch.tensor(BG, device="cuda"))
    assert not torch.equal(plain.per_view, e.per_view)
    state = tr.state_dict()
    assert state["antialiasing"] is True
    opt = lambda t: t.opt if isinstance(t, MeshTrainer) else t.adam
    fresh = _trainer(gs_type, _model(gs_type), iterations=100)
    fresh.load_state_dict(state)
    for k in ("p", "m", "v"):
        assert torch.equal(getattr(opt(fresh), k), getattr(opt(tr), k)), k
    for n in _names(gs_type):
        assert torch.equal(getattr(fresh.model, n), getattr(m, n)), n
    other = _trainer(gs_type, _model(gs_type), antialiasing=False, iterations=100)
    with pytest.raises(ValueError, match=r"antialiasing=True.*antialiasing=False"):
        other.load_state_dict(state)
    with pytest.raises(ValueError, match=r"antialiasing=False.*antialiasing=True"):
        _trainer(gs_type, _model(gs_type), iterations=100).load_state_dict(other.state_dict())


# ---------------------------------------------------------------------------------------------- 6. the default

@pytest.mark.parametrize("gs_type", TYPES)
def test_default_frames_launch_as_before(gs_type):
    """antialiasing=False (the default) draws what a frame run without the argument draws, bit for bit, and what the
    renderer draws without antialiasing; an antialiased loop issues exactly as many library launches per step as the
    default loop."""
    cams, gts = _views(gs_type, 4)
    counts = {}
    for aa in (False, True):
        m = _model(gs_type)
        tr = _trainer(gs_type, m, antialiasing=aa, iterations=100)
        for i in range(4):
            tr.step(cams[i], gts[i])
        torch.cuda.synchronize()
        _lib.launch_count(reset=True)
        for i in range(8):
            tr.step(cams[i % 4], gts[i % 4])
        torch.cuda.synchronize()
        counts[aa] = _lib.launch_count(reset=True)
    assert counts[False] == counts[True], counts
    m = _model(gs_type)
    tr = _trainer(gs_type, m, antialiasing=False)
    a = _step(tr, gs_type, cams[0], gts[0])
    fr = _frame(tr)
    fr.run(cams[0], gts[0], torch.tensor(BG, device="cuda"))
    torch.cuda.synchronize()
    b = _outputs(fr, cams[0])
    image = _renderer(gs_type, m, cams[0]).render(cams[0], torch.tensor(BG, device="cuda"))[0]
    torch.cuda.synchronize()
    assert torch.equal(a["image"], b["image"]) and torch.equal(a["radii"], b["radii"]) and torch.equal(a["image"], image)
    print(f"[{gs_type} default] library launches per 8 steps {counts}")
