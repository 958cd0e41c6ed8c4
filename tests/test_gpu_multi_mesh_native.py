"""-m gpu: gs_multi_mesh scenes with a different splat count per mesh, trained and rendered natively.

A segmented MultiMeshGaussianModel hands gms_train_frame / gms_render_frame one gms_mesh_segment (F_i, K_i) per mesh: the
unchanged expansion kernels run once per mesh at pointer offsets, everything after them once over all P Gaussians.
Checked here:
  - the frame's expansion outputs against the reference's own GaussianMultiMeshModel outputs (expansion_multi.npz);
  - four K = 5 segments against the merged single-segment model: forward bit-identical (the loss to the last bits its
    atomics leave open), gradients and the parameters after three steps within a small multiple of the run-to-run
    difference of the merged frame;
  - K = (1, 3, 40) -- one mesh too large for the staged expansion -- against the float64 oracle chain, per mesh then cat;
  - sync-free against synchronising frames under the binning / sort / compositing options, overflow and recovery;
  - NativeRenderer / evaluate() on a segmented model, and the save / load round trip of its checkpoint;
  - bad segment descriptions refused before any launch."""
import os

import numpy as np
import pytest
import torch

import aten_reference
from gms_b200 import _lib, io_ply, scenes
from gms_b200.metrics import image_metrics
from gms_b200.model import MultiMeshGaussianModel
from gms_b200.optim import REFERENCE_LRS, FlatAdam, mesh_model_groups
from gms_b200.render import NativeRenderer
from gms_b200.trainer import MeshTrainer, NativeFrame
from gms_b200.scenes import MeshGaussianParams
from gpu_helpers import GRAD_TOL, STAGE2_TOL, assert_image_parity
from helpers import settings_from_camera
from oracle import expansion as oexp
from oracle import raster
from test_gpu_native_frame import OPTION_SETS, _frame_outputs, _opt_id, _Options

pytestmark = pytest.mark.gpu

LAMBDA = 0.2
BG = (0.2, 0.5, 0.9)
W, H = 400, 300
GRADS = ("vertices", "_alpha", "_scale", "_opacity", "_features")
# the ceiling of a GPU-vs-GPU gradient difference: the backward stage tolerances (gpu_helpers.assert_backward_stages) of the
# quantities each raw parameter's gradient is formed from (vertices / _scale: through the scales and rotations; _alpha: the
# means only; opacity and SH: the per-Gaussian default)
CEILING = dict(vertices=STAGE2_TOL["scales"], _scale=STAGE2_TOL["scales"], _alpha=STAGE2_TOL["means3D"], _opacity=5e-5, _features=5e-5)
# always allowed, as max err / max|ref|: 3-5x the largest difference between two runs of the same frame measured on these
# scenes (H100: vertices 1.8e-5, _scale 3.2e-5, _alpha 2.4e-6, _opacity 2.3e-7, _features 4.3e-7).  The largest element of the
# atomics' summation noise varies by 30x from one pair of runs to the next, so one pair alone is no yardstick.
NOISE = dict(vertices=1e-4, _scale=1e-4, _alpha=1e-5, _opacity=1e-6, _features=1e-6)
# the same for the parameters after three Adam steps (measured: _alpha 1.2e-6, _scale 3.6e-6, _opacity 9.3e-7, _features 1e-7;
# the vertices' learning rate is 0)
PARAM_NOISE = dict(vertices=1e-6, _alpha=1e-5, _scale=2e-5, _opacity=5e-6, _features=1e-6)


def _meshes(Ks, levels, seed=0):
    """Disjoint meshes side by side along x, mesh k with K = Ks[k] splats per face."""
    plist = []
    for k, (K, lvl) in enumerate(zip(Ks, levels)):
        v, f = scenes.icosphere(lvl, radius=0.35 + 0.05 * k)
        p = scenes.init_mesh_gaussians(v + np.float32([0.8 * k - 0.4 * (len(Ks) - 1), 0.1 * k, 0]), f, K=K, seed=seed + k,
                                       trained_like=True)
        p._scale = 0.6 + 0.8 * torch.rand(p._scale.shape, generator=torch.Generator().manual_seed(100 + seed + k))
        plist.append(p)
    return plist


def _camera():
    return scenes.look_at_camera((0.4, 1.2, 2.6), (0.0, 0.0, 0.0), W, H)


def _gt():
    return torch.rand(3, H, W, generator=torch.Generator().manual_seed(W * H))


def _model(plist, segmented=False):
    return MultiMeshGaussianModel.from_mesh_params(plist, "cuda", packed_features=True, segmented=segmented)


def _frame(plist, segmented=False, sync_free=True, **opt_kw):
    m = _model(plist, segmented)
    opt = FlatAdam(mesh_model_groups(m, features_last=opt_kw.get("sh_factored", False)), **opt_kw)
    return m, opt, NativeFrame(m, W, H, LAMBDA, sync_free=sync_free)


def _run(fr, opt, cam, gt, bg):
    opt.zero_grad()
    loss = fr.run(cam, gt, bg).item()
    torch.cuda.synchronize()
    return loss


def _grads(m):
    return {k: getattr(m, k).grad.detach().clone() for k in GRADS}


def _rel(a, b):
    a, b = a.reshape(-1).double(), b.reshape(-1).double()        # (merged _alpha is [F,K,3], segmented [P,3]: same order)
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)


def _same_loss(a, b):
    """The loss kernels add their per-block partial sums with float atomics, so two runs on the same image may differ in the
    last bits of the loss: allowed 1e-6 relative (measured: 3 ulp)."""
    return abs(a - b) <= 1e-6 * abs(b)


def _assert_within_run_to_run(got, ref, ref2, what, ceiling=CEILING):
    """Each tensor of `got` agrees with `ref` within 8x the difference between `ref` and `ref2` (two runs of the reference
    arm) or NOISE, whichever is larger, never above the ceiling."""
    msg = []
    for k in ref:
        e, e0 = _rel(got[k], ref[k]), _rel(ref2[k], ref[k])
        msg.append(f"{k} {e:.1e} (run-to-run {e0:.1e})")
        assert e <= min(ceiling[k], max(8.0 * e0, NOISE[k])), (what, k, e, e0)
    print(f"[multi-mesh] {what}: " + ", ".join(msg))


def test_frame_expansion_matches_reference_golden(golden_dir):
    """expansion_multi.npz (the reference's GaussianMultiMeshModel, K = 2 and 3): the training frame's activated expansion
    outputs (gms_frame_views) equal the reference's, at the tolerances of test_gpu_expansion's multi-mesh test."""
    g = np.load(os.path.join(golden_dir, "expansion_multi.npz"))
    plist = []
    for k in range(int(g["n_mesh"])):
        a, s = torch.tensor(g[f"_alpha{k}"]), torch.tensor(g[f"_scale{k}"])
        P = s.shape[0]
        gen = torch.Generator().manual_seed(k)
        plist.append(MeshGaussianParams(torch.tensor(g[f"vertices{k}"]), torch.tensor(g[f"faces{k}"]).long(), a, s,
                                        torch.randn(P, 1, 3, generator=gen), 0.05 * torch.randn(P, 15, 3, generator=gen),
                                        torch.randn(P, 1, generator=gen)))
    m, opt, fr = _frame(plist)
    assert m.segments == [(20, 2), (80, 3)]
    cam = scenes.look_at_camera((0.75, 1.0, 3.0), (0.75, 0.0, 0.0), W, H).to("cuda")
    _run(fr, opt, cam, _gt().cuda(), torch.tensor(BG, device="cuda"))
    out = _frame_outputs(fr, m._scale.shape[0])
    np.testing.assert_allclose(out["xyz"].numpy(), g["xyz"], atol=1e-6)
    np.testing.assert_allclose(np.log(out["scales"].numpy()), g["_scaling"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(out["rotations"].numpy(), torch.nn.functional.normalize(torch.tensor(g["_rotation"])).numpy(), atol=1e-6)


def test_equal_k_segments_match_the_merged_model():
    """Four K = 5 meshes as four segments against the merged single-segment model with the same parameters."""
    plist = _meshes((5, 5, 5, 5), (3, 3, 3, 3), seed=3)
    cam, gt, bg = _camera().to("cuda"), _gt().cuda(), torch.tensor(BG, device="cuda")
    runs = {}
    for name, seg in (("merged", False), ("merged2", False), ("segmented", True)):
        m, opt, fr = _frame(plist, seg)
        assert (m.segments is not None) == seg
        _run(fr, opt, cam, gt, bg)                       # synchronising: learns N
        loss = _run(fr, opt, cam, gt, bg)                # sync-free
        runs[name] = (loss, fr.last_num_rendered, _frame_outputs(fr, m._scale.shape[0]), _grads(m))
    lm, nm, om, gm = runs["merged"]
    ls, ns, os_, gs = runs["segmented"]
    assert _same_loss(ls, lm) and ns == nm
    for k in om:
        assert torch.equal(os_[k], om[k]), k
    _assert_within_run_to_run(gs, gm, runs["merged2"][3], "gradients, 4 segments vs merged")


@pytest.mark.parametrize("factored", [False, True], ids=["fused_sh_adam", "factored"])
def test_equal_k_segments_train_like_the_merged_model(factored):
    """The parameters after three steps: MeshTrainer (native, the SH Adam fused into the frame), or NativeFrame(factored=True)
    with FlatAdam's factored SH step."""
    plist = _meshes((5, 5, 5, 5), (3, 3, 3, 3), seed=5)
    cams = [c.to("cuda") for c in scenes.ring_cameras(3, 2.6, W, H)]
    gt, bg = _gt().cuda(), torch.tensor(BG, device="cuda")
    params = {}
    for name, seg in (("merged", False), ("merged2", False), ("segmented", True)):
        if not factored:
            m = _model(plist, seg)
            tr = MeshTrainer(m, bg, LAMBDA, native=True)
            for c in cams:
                tr.step(c, gt)
        else:
            m, opt, fr = _frame(plist, seg, sh_factored=True)
            for c in cams:
                fr.run(c, gt, bg, factored=True)
                opt.step(zero_end=opt.ends[0], sh=fr.sh_factors())
        torch.cuda.synchronize()
        params[name] = {k: getattr(m, k).detach().clone() for k in GRADS}
    _assert_after_steps(params["segmented"], params["merged"], params["merged2"], "params after 3 steps" + (", factored" if factored else ""))


def _assert_after_steps(got, ref, ref2, what):
    """As _assert_within_run_to_run, for parameters after Adam steps.  Adam's first step moves every element by lr * sign(g):
    an element whose gradient is at the level of the atomics' summation noise may take the other sign in another run (a
    change of 2 lr).  Elements that moved by more than lr / 2 are counted -- at most 4 more than between the two reference
    runs -- and left out of the comparison."""
    lr = dict(vertices=REFERENCE_LRS["vertices"], _alpha=REFERENCE_LRS["alpha"], _scale=REFERENCE_LRS["scaling"],
              _opacity=REFERENCE_LRS["opacity"], _features=REFERENCE_LRS["f_rest"])       # (the smallest rate of the group)
    msg = []
    for k in ref:
        g, r, r2 = got[k].reshape(-1), ref[k].reshape(-1), ref2[k].reshape(-1)
        d, d0 = (g - r).abs(), (r2 - r).abs()
        flip, flip0 = d > 0.5 * lr[k], d0 > 0.5 * lr[k]
        assert int(flip.sum()) <= int(flip0.sum()) + 4, (what, k, int(flip.sum()), int(flip0.sum()))
        scale = max(float(r.abs().max()), 1e-30)
        e, e0 = float(d[~flip].max()) / scale if (~flip).any() else 0.0, float(d0[~flip0].max()) / scale if (~flip0).any() else 0.0
        msg.append(f"{k} {e:.1e} (run-to-run {e0:.1e}, sign flips {int(flip.sum())}/{int(flip0.sum())})")
        assert e <= max(8.0 * e0, PARAM_NOISE[k]), (what, k, e, e0)
    print(f"[multi-mesh] {what}: " + ", ".join(msg))


# K = 1 and 3 take the staged expansion; K = 40 exceeds its 48 KB of shared memory and runs the direct kernel
HETERO = dict(Ks=(1, 3, 40), levels=(3, 3, 1))


def _oracle_segmented(plist, S, dC, out):
    """Oracle chain of a segmented scene: oracle/expansion.py in float64 per mesh on the merged vertices, concatenated; the
    oracle rasterizer on the Gaussians the GPU frame drew (so that integer outputs compare bit for bit), its backward chained
    through the float64 expansion graph.  -> (state, gradients of the flat raw parameters)."""
    m = MultiMeshGaussianModel.from_mesh_params(plist, "cpu")
    tv, ta, ts, top = (getattr(m, k).detach().double().requires_grad_(True) for k in ("vertices", "_alpha", "_scale", "_opacity"))
    xyz, sl, rr, f0, g0 = [], [], [], 0, 0
    for F, K in m.segments:
        x, s, r, _, _ = oexp.expand(tv, m.faces[f0:f0 + F], ta[g0:g0 + F * K].view(F, K, 3), ts[g0:g0 + F * K])
        xyz.append(x); sl.append(s); rr.append(r)
        f0, g0 = f0 + F, g0 + F * K
    xyz, sl, rr = torch.cat(xyz), torch.cat(sl), torch.cat(rr)
    sc, rot, op = torch.exp(sl), torch.nn.functional.normalize(rr), torch.sigmoid(top)
    gx, gs, gr = out["xyz"], out["scales"], out["rotations"]
    # q and -q are the same rotation; on faces where the fp32 and float64 quaternion branches differ (symmetric meshes) they
    # are of opposite sign, and the rasterizer's gradient for the GPU's q enters the float64 graph with that sign
    sgn = torch.where((gr.double() * rot.detach()).sum(1, keepdim=True) < 0, -1.0, 1.0).double()
    assert float((gx.double() - xyz.detach()).abs().max()) <= 2e-6 and float((gr.double() - sgn * rot.detach()).abs().max()) <= 4e-6
    assert float(((gs.double() - sc.detach()).abs() / sc.detach()).max()) <= 1e-5
    print(f"[multi-mesh] quaternions of opposite sign in fp32 and float64: {int((sgn < 0).sum())} of {sgn.shape[0]}")
    fe = m.get_features.detach()
    st = raster.forward(S, gx, torch.sigmoid(m._opacity.detach()), shs=fe.contiguous(), scales=gs, rotations=gr)
    g = raster.backward(st, dC)
    up = {k: torch.tensor(g[k], dtype=torch.float64).reshape(t.shape) for k, t in
          (("dL_dmeans3D", xyz), ("dL_dscales", sc), ("dL_drotations", rot), ("dL_dopacity", op))}
    torch.autograd.backward([xyz, sc, rot, op], [up["dL_dmeans3D"], up["dL_dscales"], sgn * up["dL_drotations"], up["dL_dopacity"]])
    return st, dict(vertices=tv.grad, _alpha=ta.grad, _scale=ts.grad, _opacity=top.grad,
                    _features=torch.tensor(g["dL_dsh"]).reshape(fe.shape))


def test_heterogeneous_k_frame_matches_oracle():
    """K = (1, 3, 40), the first sync-free frame: radii and N bit-exact, image within 1e-5 outside the threshold-ambiguous
    pixels, loss, and every raw-parameter gradient at the reference-render tolerances."""
    plist = _meshes(**HETERO, seed=11)
    cam, gt = _camera(), _gt()
    m, opt, fr = _frame(plist)
    assert m.segments == [(1280, 1), (1280, 3), (80, 40)]
    cam_d, gt_d, bg = cam.to("cuda"), gt.cuda(), torch.tensor(BG, device="cuda")
    _run(fr, opt, cam_d, gt_d, bg)
    n_first = fr.last_num_rendered
    loss = _run(fr, opt, cam_d, gt_d, bg)
    assert fr.overflows == 0 and fr.capacity > n_first > 0
    out = _frame_outputs(fr, m._scale.shape[0])
    img = out["image"].double().requires_grad_(True)
    aten_reference.training_loss(img, gt.double(), LAMBDA).backward()
    st, og = _oracle_segmented(plist, settings_from_camera(cam, bg=BG), img.grad.float().numpy(), out)
    np.testing.assert_array_equal(out["radii"].numpy(), st.radii)
    assert fr.last_num_rendered == st.N
    assert_image_parity(st, out["image"].numpy())
    with torch.no_grad():
        ref_loss = float(aten_reference.training_loss(torch.tensor(st.color, dtype=torch.float64), gt.double(), LAMBDA))
    assert abs(loss - ref_loss) <= 1e-5 * max(1.0, abs(ref_loss))
    msg = []
    for k, ref_g in og.items():
        e = _rel(getattr(m, k).grad.detach().cpu().reshape(ref_g.shape), ref_g)
        msg.append(f"{k} {e:.2e}")
        assert e <= GRAD_TOL.get(k, 2e-4), (k, e)
    print(f"[multi-mesh] K=(1,3,40) P={m._scale.shape[0]} N={st.N} vs oracle, grad max err / max|ref|: " + ", ".join(msg))


@pytest.mark.parametrize("opts", OPTION_SETS, ids=_opt_id)
def test_heterogeneous_k_sync_free_equals_synchronising(opts):
    """The same heterogeneous frame synchronising (capacity = N) and sync-free (predicted capacity): radii, N and image
    bit-identical, the loss to the last bits its atomics leave open; gradients within the run-to-run difference of the
    synchronising frame."""
    plist = _meshes(**HETERO, seed=13)
    cam, gt, bg = _camera().to("cuda"), _gt().cuda(), torch.tensor(BG, device="cuda")
    res = {}
    with _Options(opts):
        for name, sync_free in (("sync", False), ("sync2", False), ("free", True)):
            m, opt, fr = _frame(plist, sync_free=sync_free)
            _run(fr, opt, cam, gt, bg)
            loss = _run(fr, opt, cam, gt, bg)
            assert fr.capacity > 0 if sync_free else fr.capacity == 0
            res[name] = (loss, fr.last_num_rendered, _frame_outputs(fr, m._scale.shape[0]), _grads(m))
    (l0, n0, o0, g0), (l1, n1, o1, g1) = res["sync"], res["free"]
    assert _same_loss(l1, l0) and n1 == n0
    for k in ("radii", "image", "invdepth"):
        assert torch.equal(o1[k], o0[k]), k
    _assert_within_run_to_run(g1, g0, res["sync2"][3], "sync-free vs synchronising, " + _opt_id(opts))


def test_heterogeneous_k_overflow_renders_background_then_recovers():
    plist = _meshes(**HETERO, seed=13)
    cam, gt, bg = _camera().to("cuda"), _gt().cuda(), torch.tensor(BG, device="cuda")
    _, sopt, sfr = _frame(plist, sync_free=False)
    _run(sfr, sopt, cam, gt, bg)
    ref = _frame_outputs(sfr, sfr.model._scale.shape[0])
    m, opt, fr = _frame(plist)
    _run(fr, opt, cam, gt, bg)
    N = fr.last_num_rendered
    fr.capacity_override = N - 1
    _run(fr, opt, cam, gt, bg)
    assert fr.last_num_rendered == N and fr.overflows == 1
    out = _frame_outputs(fr, m._scale.shape[0])
    assert torch.equal(out["image"], torch.tensor(BG)[:, None, None].expand(3, H, W))
    assert float(out["invdepth"].abs().max()) == 0.0
    for k in GRADS:
        assert float(getattr(m, k).grad.abs().max()) == 0.0, k
    fr.capacity_override = None
    _run(fr, opt, cam, gt, bg)
    assert fr.overflows == 1 and fr.capacity > N
    out = _frame_outputs(fr, m._scale.shape[0])
    for k in ("radii", "image", "invdepth"):
        assert torch.equal(out[k], ref[k]), k


def test_renderer_and_evaluate_on_a_segmented_model():
    """NativeRenderer draws a segmented model bit-identically to the training frame's forward (first, synchronising render
    and the sync-free ones after it); evaluate() scores it as a per-view render + image_metrics does."""
    plist = _meshes(**HETERO, seed=17)
    cams = [c.to("cuda") for c in scenes.ring_cameras(3, 2.6, W, H)]
    gts = [torch.rand(3, H, W, generator=torch.Generator().manual_seed(i)).cuda() for i in range(3)]
    bg = torch.tensor(BG, device="cuda")
    m, opt, fr = _frame(plist, sync_free=False)
    r = NativeRenderer(m, W, H)
    for rep in range(2):
        for c, gt in zip(cams, gts):
            _run(fr, opt, c, gt, bg)
            ref = _frame_outputs(fr, m._scale.shape[0])
            img, radii, invd = r.render(c, bg)
            for k, t in (("image", img), ("radii", radii), ("invdepth", invd)):
                assert torch.equal(t.cpu(), ref[k]), (rep, k)
    assert r.capacity > 0 and r.overflows == 0
    res = r.evaluate(cams, gts, bg)
    for v, (c, gt) in enumerate(zip(cams, gts)):
        r.render(c, bg)
        want = image_metrics(r.image, gt, "training_report").cpu()
        assert torch.equal(res.per_view[v], want), v
    tr = MeshTrainer(m, bg, LAMBDA, native=True)
    assert torch.equal(tr.evaluate(cams, gts).per_view, res.per_view)


def test_checkpoint_round_trip(tmp_path):
    """save_multi_mesh_model -> load_multi_mesh_model gives back every tensor exactly; the PLY's Gaussians are the
    per-mesh expansion's, in the reference's cat order."""
    plist = _meshes(**HETERO, seed=19)
    m = _model(plist)
    ply = str(tmp_path / "point_cloud.ply")
    io_ply.save_multi_mesh_model(ply, m)
    back = io_ply.load_multi_mesh_model(ply)
    assert len(back) == len(plist)
    for p, q in zip(plist, back):
        for k in ("vertices", "faces", "_alpha", "_scale", "_features_dc", "_features_rest", "_opacity"):
            assert torch.equal(getattr(q, k), getattr(p, k).to(getattr(q, k).dtype)), k
    xyz, sl, rr = MultiMeshGaussianModel.expand_per_mesh([p.vertices.cuda() for p in plist], [p.faces.cuda() for p in plist],
                                                         [p._alpha.cuda() for p in plist], [p._scale.cuda() for p in plist])
    g = io_ply.load_gaussian_ply(ply)       # written through update_alpha / prepare_scaling_rot, the reference's two-step protocol
    np.testing.assert_allclose(g["_xyz"].numpy(), xyz.cpu().numpy(), atol=1e-6)
    np.testing.assert_allclose(g["_scaling"].numpy(), sl.cpu().numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(g["_rotation"].numpy(), rr.cpu().numpy(), atol=1e-6)
    m2 = MultiMeshGaussianModel.from_mesh_params(back, "cuda", packed_features=True)
    assert m2.segments == m.segments and torch.equal(m2._alpha, m._alpha) and torch.equal(m2._features, m._features)


def test_bad_segments_are_refused_before_any_launch():
    """A wrong sum of F, K != 0 with segments, K_i = 0, P above int32 and a too-small workspace: GMS_E_ARG from both
    gms_train_frame and gms_render_frame, and the library issued no launch."""
    plist = _meshes(**HETERO, seed=23)
    cam, gt, bg = _camera().to("cuda"), _gt().cuda(), torch.tensor(BG, device="cuda")
    m, opt, fr = _frame(plist, sync_free=False)
    r = NativeRenderer(m, W, H)
    F = m.faces.shape[0]
    bad = {"sum of F": (F, 0, [(1281, 1), (1280, 3), (80, 40)]), "K != 0": (F, 3, m.segments),
           "K_i = 0": (F, 0, [(1280, 1), (1280, 0), (80, 40)]), "P overflow": (F, 0, [(1280, 1 << 21), (1280, 3), (80, 40)])}
    for what, (F_, K_, seg) in bad.items():
        arr = _lib.mesh_segments(seg)
        m.frame_sizes = lambda: (F_, K_, arr)
        for call in (lambda: fr.run(cam, gt, bg), lambda: r.render(cam, bg)):
            n0 = _lib.launch_count()
            with pytest.raises(Exception, match="segment|K must be 0|int32|F must equal"):
                call()
            assert _lib.launch_count() == n0, what
    del m.frame_sizes
    ws, fr.ws = fr.ws, fr.ws[:fr.ws.numel() // 2]
    rws, r.ws = r.ws, r.ws[:r.ws.numel() // 2]
    for call in (lambda: fr.run(cam, gt, bg), lambda: r.render(cam, bg)):
        n0 = _lib.launch_count()
        with pytest.raises(Exception, match="workspace too small"):
            call()
        assert _lib.launch_count() == n0
    fr.ws, r.ws = ws, rws
    fr.run(cam, gt, bg)         # the same objects, with the right sizes, run
    r.render(cam, bg)
    torch.cuda.synchronize()
