"""-m gpu: training on views of different sizes, for gs_mesh, segmented gs_multi_mesh, gs_flame, gs and gs_flat.

A trainer's one frame is sized for the largest view and runs every view at the view's own size.  Checked here: a view run
in a frame sized for a larger one is the exact-size frame (image, radii and inverse depth bit for bit; the loss and the
gradients within the spread of the float atomics that sum them); a training loop over alternating sizes agrees with a
loop that gives each size an exact-size frame over the same model and optimizer, and never synchronises after each
view's first frame; gs / gs_flat keep running on every size as densification changes P; evaluate() over a mixed split is
the per-size renders; and cli.train trains, saves and resumes on a mixed-size scene that cli.render and cli.metrics then
read."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import mesh_types_cases
import mixed_sizes_cases as cases
from gms_b200 import _lib, dataset, io_image, scenes
from gms_b200.cli import metrics as cli_metrics
from gms_b200.cli import render as cli_render
from gms_b200.cli import train as cli_train
from gms_b200.flame import NativeFlame
from gms_b200.model import FlameGaussianModel, FreeGaussianModel, MeshGaussianModel, MultiMeshGaussianModel
from gms_b200.render import NativeFreeRenderer, NativeRenderer
from gms_b200.trainer import (FlameOptimizationParams, FlameTrainer, FreeOptimizationParams, FreeTrainer, MeshTrainer,
                              NativeFrame, NativeFreeFrame)
from helpers import random_gaussians

pytestmark = pytest.mark.gpu

TYPES = ["gs_mesh", "gs_multi_mesh", "gs_flame", "gs", "gs_flat"]
MESH_TYPES = ("gs_mesh", "gs_multi_mesh")
LAMBDA = 0.2
BG = (0.2, 0.5, 0.9)
LAND, PORT = (256, 144), (144, 256)         # ragged tile grids (144 = 9 tiles, 256 = 16)
MAX = (256, 256)
# the sync-free / atomics spread bound of the frame tests (DESIGN.md 4.3, test_gpu_free_train.SYNC_NOISE), max |diff| /
# max |grad| per tensor; mesh vertices, alpha and the FLAME tensors gather the scale and rotation gradients, so they get
# the scaling bound
SYNC_NOISE = {"_xyz": 1.5e-4, "_scaling": 4e-3, "_rotation": 1.5e-3, "_opacity": 1e-6, "_features": 1e-6}
MESH_NOISE = {"vertices": 4e-3, "_alpha": 4e-3, "_scale": 4e-3, "_scales": 4e-3, "_opacity": 1e-6, "_features": 1e-6}


def _names(gs_type):
    if gs_type in MESH_TYPES:
        return ("vertices", "_alpha", "_scale", "_features", "_opacity")
    if gs_type == "gs_flame":
        return FlameGaussianModel.FLAME_NAMES + ("_alpha", "_scales", "_features", "_opacity")
    return FreeGaussianModel.NAMES


def _bound(name):
    return SYNC_NOISE.get(name, MESH_NOISE.get(name, 4e-3))


def _model(gs_type):
    if gs_type == "gs_mesh":
        return MeshGaussianModel.from_params(scenes.init_mesh_gaussians(*scenes.icosphere(3, 0.8), K=3, seed=1), "cuda",
                                             packed_features=True)
    if gs_type == "gs_multi_mesh":
        v0, f0 = scenes.icosphere(2, 0.7)
        v1, f1 = scenes.icosphere(1, 0.35)
        p = [scenes.init_mesh_gaussians(v0, f0, K=2, seed=2), scenes.init_mesh_gaussians(v1 + np.array([0.5, -0.2, 0.3]), f1, K=5, seed=3)]
        m = MultiMeshGaussianModel.from_mesh_params(p, "cuda", packed_features=True)
        assert m.segments is not None
        return m
    if gs_type == "gs_flame":
        init = dataset.flame_init(mesh_types_cases.FLAME_MODEL)
        return FlameGaussianModel.create(NativeFlame.from_model_file(mesh_types_cases.FLAME_MODEL), init.faces, K=60, seed=4)
    g = random_gaussians(3000, seed=5, extent=0.8, flat_frac=0.0)
    s = torch.log(g["scales"])
    return FreeGaussianModel(g["means3D"], (s[:, 1:] if gs_type == "gs_flat" else s).contiguous(), g["rotations"], g["shs"],
                             torch.logit(g["opacities"]), gs_type, "cuda", 3)


def _trainer(gs_type, model, max_size, iterations=1000, **free):
    bg = torch.tensor(BG, device="cuda")
    if gs_type in MESH_TYPES:
        return MeshTrainer(model, bg, LAMBDA, native=True, max_size=max_size)
    if gs_type == "gs_flame":
        return FlameTrainer(model, bg, FlameOptimizationParams(iterations=iterations), max_size=max_size)
    return FreeTrainer(model, bg, 1.0, FreeOptimizationParams(iterations=iterations, **free), max_size=max_size)


def _frame(tr):
    return tr._frame if isinstance(tr, MeshTrainer) else tr.frame


def _set_frame(tr, fr):
    if isinstance(tr, MeshTrainer):
        tr._frame = fr
    else:
        tr.frame = fr


def _views(n=4, seed=0):
    """n cameras around the origin alternating landscape and portrait, with uint8 ground truth of their sizes."""
    cams, gts = [], []
    g = torch.Generator().manual_seed(seed)
    for k in range(n):
        W, H = (LAND, PORT)[k % 2]
        c = scenes.ring_cameras(n, 2.6, W, H, phase=0.3)[k]
        c.uid = ("view", k)
        cams.append(c.to("cuda"))
        gts.append(torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8).cuda())
    return cams, gts


def _outputs(fr, cam):
    """The frame's radii, image and inverse depth at `cam`'s size (gms_frame_views), and its loss vector."""
    P = fr._gaussians()
    W, H = int(cam.image_width), int(cam.image_height)
    v = _lib.FrameView()
    _lib.check(_lib.lib().gms_frame_views(fr.ws.data_ptr(), P, W, H, C.byref(v)), "gms_frame_views")

    def take(ptr, shape, dtype=torch.float32):
        off = ptr - fr.ws.data_ptr()
        return fr.ws[off:off + 4 * int(np.prod(shape))].view(dtype).view(shape).clone()

    return dict(radii=take(v.radii, (P,), torch.int32), image=take(v.image, (3, H, W)), invdepth=take(v.invdepth, (1, H, W)),
                loss=fr.loss.clone())


def _step(tr, gs_type, cam, gt):
    """One step with a before_update hook that copies the frame's gradients (the step takes no Adam step here)."""
    grads = {}

    def grab():
        for n in _names(gs_type):
            grads[n] = getattr(tr.model, n).grad.detach().clone()

    tr.step(cam, gt, before_update=grab)
    torch.cuda.synchronize()
    out = _outputs(_frame(tr), cam)
    out["grads"] = grads
    return out


def _rel(a, b):
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-20)


@pytest.mark.parametrize("gs_type", TYPES)
def test_small_view_in_large_frame_is_the_exact_size_frame(gs_type):
    """A landscape view run (sync-free, after a portrait one) in a frame sized for 256x256 against the same view's second
    frame in a frame sized for it: image, radii and inverse depth bit for bit; gradients within the spread bound.  The loss
    kernels add their per-block partial sums of L1 and SSIM with float atomics, so two runs of one frame may already differ
    in the last bits of the loss: it is held to 2e-6 relative, against a bit-identical image."""
    cams, gts = _views(2)
    big_m, exact_m = _model(gs_type), _model(gs_type)
    big, exact = _trainer(gs_type, big_m, MAX, iterations=1), _trainer(gs_type, exact_m, None, iterations=1)
    if gs_type in MESH_TYPES:
        big.optimizer_step = exact.optimizer_step = False       # no Adam step (the others take none at iterations=1)
    _step(big, gs_type, cams[1], gts[1])
    b = _step(big, gs_type, cams[0], gts[0])
    a1 = _step(exact, gs_type, cams[0], gts[0])
    a2 = _step(exact, gs_type, cams[0], gts[0])
    fb, fa = _frame(big), _frame(exact)
    assert (fb.W, fb.H, fb.up_to) == (*MAX, True) and (fa.W, fa.H) == LAND
    assert fb.overflows == 0 and fa.overflows == 0 and fb.capacity > 0
    assert int((a2["radii"] > 0).sum()) > 100, "the view must see the model"
    for k in ("radii", "image", "invdepth"):
        assert torch.equal(b[k], a2[k]), k
        assert torch.equal(a1[k], a2[k]), k
    for x in (b, a1):
        assert bool(((x["loss"] - a2["loss"]).abs() <= 2e-6 * a2["loss"].abs()).all()), (x["loss"].tolist(), a2["loss"].tolist())
    msg = []
    for n in _names(gs_type):
        spread, got = _rel(a1["grads"][n], a2["grads"][n]), _rel(b["grads"][n], a2["grads"][n])
        msg.append(f"{n} {got:.1e} (run-to-run {spread:.1e})")
        assert got <= max(_bound(n), 10 * spread), (n, got, spread)
    print(f"[{gs_type} small in large] grad |diff| / max|grad|: " + ", ".join(msg))


FREE_TYPES = ("gs", "gs_flat")
N_LOOP = 48


def _exact_frame(tr, gs_type, cam):
    W, H = int(cam.image_width), int(cam.image_height)
    if gs_type in FREE_TYPES:
        return NativeFreeFrame(tr.model, W, H, LAMBDA)
    return NativeFrame(tr.model, W, H, LAMBDA)


def _loop(gs_type, mode, strict=False):
    """N_LOOP steps over four views alternating landscape and portrait, Adam on.  mode "max": max_size given; "grow": sized
    from the first view and grown; "exact": one exact-size frame per size swapped in before each step.  strict: every
    frame but each view's first runs under sync debug mode "error".  -> the losses [N_LOOP]."""
    cams, gts = _views(4)
    m = _model(gs_type)
    tr = _trainer(gs_type, m, MAX if mode == "max" else None, iterations=N_LOOP)
    frames, seen, losses = {}, set(), []
    try:
        for it in range(N_LOOP):
            v = it % 4
            if mode == "exact":
                size = (cams[v].image_width, cams[v].image_height)
                if size not in frames:
                    frames[size] = _exact_frame(tr, gs_type, cams[v])
                _set_frame(tr, frames[size])
            if strict:
                torch.cuda.set_sync_debug_mode(0 if v not in seen else "error")
            seen.add(v)
            losses.append(tr.step(cams[v], gts[v]).clone())
    finally:
        torch.cuda.set_sync_debug_mode(0)
    fr = _frame(tr)
    if mode != "exact":
        assert (fr.W, fr.H) == MAX and fr.overflows == 0
    return torch.stack(losses).cpu().double()


@pytest.mark.parametrize("gs_type", TYPES)
def test_mixed_loop_matches_exact_size_frames(gs_type):
    """The loop over alternating sizes (one frame for the largest view, and one grown from the first view) against the
    loop with an exact-size frame per size: every iteration's loss within 10x the mixed loop's own run-to-run spread (plus
    1e-5 of the loss); the mixed loop never synchronises after each view's first frame."""
    la = _loop(gs_type, "max", strict=True)
    lb = _loop(gs_type, "max")
    for mode in ("exact", "grow"):
        lr = _loop(gs_type, mode)
        d, spread = float((lr - la).abs().max()), float((lb - la).abs().max())
        print(f"[{gs_type} {mode}] losses: max |diff| {d:.3e}, run-to-run {spread:.3e}")
        assert d <= 10 * spread + 1e-5 * float(la.abs().max()), (mode, d, spread)
    assert bool(torch.isfinite(la).all())


@pytest.mark.parametrize("gs_type", FREE_TYPES)
def test_densification_keeps_every_size_running(gs_type):
    """Densify every 8 iterations from iteration 4 over alternating sizes: P changes, the frame keeps the largest size,
    every size runs after each change, no frame overflows and every loss is finite."""
    cams, gts = _views(4)
    m = _model(gs_type)
    P0 = m.P
    tr = _trainer(gs_type, m, MAX, iterations=60, densify_from_iter=4, densification_interval=8, densify_until_iter=60,
                  densify_grad_threshold=1e-6)
    losses = [tr.step(cams[it % 4], gts[it % 4]).clone() for it in range(60)]
    fr = tr.frame
    assert len(tr.densifications) >= 5 and m.P != P0
    assert tr.densifications[-1][0] <= 56, "both sizes run after the last densification"
    assert (fr.W, fr.H) == MAX and fr.up_to and fr.accum.shape[0] == m.P and fr.overflows == 0
    assert bool(torch.isfinite(torch.stack(losses)).all())
    print(f"[{gs_type} densify] P {P0} -> {m.P} over {len(tr.densifications)} densifications")


@pytest.mark.parametrize("gs_type", TYPES)
def test_evaluate_over_mixed_sizes_is_the_per_size_renders(gs_type):
    """evaluate() over landscape and portrait views: per view, the metrics of a renderer of that view's size, bit for bit and
    in view order; the means are those values averaged in float64; trainer.renderer draws each view at its size."""
    cams, gts = _views(5, seed=3)
    m = _model(gs_type)
    tr = _trainer(gs_type, m, MAX)
    tr.step(cams[0], gts[0])
    e = tr.evaluate(cams, gts)
    cls = NativeFreeRenderer if gs_type in FREE_TYPES else NativeRenderer
    bg = torch.tensor(BG, device="cuda")
    rows = []
    for c, g in zip(cams, gts):
        r = cls(m, c.image_width, c.image_height)
        rows.append(r.evaluate([c], [g], bg).per_view[0])
        image = tr.renderer.render(c, bg)[0]
        assert tuple(image.shape) == (3, c.image_height, c.image_width)
        assert torch.equal(image, r.render(c, bg)[0])
    want = torch.stack(rows)
    assert e.rerun == [] and torch.equal(e.per_view, want)
    assert torch.equal(e.mean, want.mean(0)) and e.mean.dtype == torch.float64
    print(f"[{gs_type} evaluate] mean {e.mean.tolist()}")


# ------------------------------------------------------------------------------------------------ the command line

N_CLI = 20
COMMON = ["--eval", "--iterations", str(N_CLI), "--test_iterations", "10", "--save_iterations", "10", "--checkpoint_iterations",
          "12", "--quiet"]


def _argv(gs_type):
    if gs_type == "gs_multi_mesh":
        return ["--gs_type", gs_type, "--meshes", *cases.MESHES, "--num_splats", *map(str, cases.NUM_SPLATS)] + COMMON
    if gs_type == "gs_flame":
        return ["--gs_type", gs_type, "--flame_model", mesh_types_cases.FLAME_MODEL] + COMMON
    return ["--gs_type", gs_type] + COMMON


@pytest.fixture(scope="module")
def roots(tmp_path_factory):
    base = tmp_path_factory.mktemp("mixed_cli")
    return {"blender": cases.write_blender(str(base / "blender")), "colmap": cases.write_colmap(str(base / "colmap"))}


def _cli(root, out, gs_type, extra=()):
    return cli_train.Training(cli_train.parse_args(["-s", root, "-m", out] + _argv(gs_type) + list(extra))).prepare()


@pytest.mark.parametrize("gs_type", TYPES)
def test_cli_trains_resumes_renders_and_scores_a_mixed_size_scene(roots, gs_type, tmp_path):
    root = roots["colmap" if gs_type == "gs_multi_mesh" else "blender"]
    out = str(tmp_path / "a")
    a = _cli(root, out, gs_type).run()
    sizes = {(c.image_width, c.image_height) for c in a.scene.train_cameras}
    assert len(sizes) == 2 and {(c.image_width, c.image_height) for c in a.scene.test_cameras} == sizes
    fr = _frame(a.trainer)
    assert (fr.W, fr.H) == cli_train.training_size(a.scene) == (48, 48) and fr.overflows == 0
    assert [(it, s) for it, s, _, _ in a.reports] == [(10, "test"), (10, "train")]
    assert all(np.isfinite(l1) and np.isfinite(psnr) for _, _, l1, psnr in a.reports)
    assert [it for it, _, _ in a.ema] == list(range(1, N_CLI + 1)) and all(np.isfinite(l) for _, l, _ in a.ema)
    for it in (10, N_CLI):
        assert os.path.exists(os.path.join(out, "point_cloud", f"iteration_{it}", "point_cloud.ply"))
    names = _names(gs_type)
    final_a = {n: getattr(a.model, n).detach().clone() for n in names}
    b = _cli(root, str(tmp_path / "b"), gs_type).run()
    final_b = {n: getattr(b.model, n).detach().clone() for n in names}
    ck = os.path.join(out, "chkpnt12.pth")
    state, k = torch.load(ck, map_location="cpu", weights_only=True)
    c = _cli(root, str(tmp_path / "c"), gs_type, ["--start_checkpoint", ck])
    now = c.trainer.state_dict()
    for key in ("p", "m", "v"):
        assert torch.equal(now["adam"][key].cpu(), state["trainer"]["adam"][key]), key
    assert k == 12 and c.first_iter == 12 and c.order.state_dict() == state["view_order"]
    c.run()
    assert [it for it, _ in c.events] == list(range(13, N_CLI + 1))
    # the resumed run starts from the checkpoint's state bit for bit; from there its frames sum with float atomics in their
    # own order, as a second uninterrupted run's do.  One pair of runs can agree exactly in a tensor by chance (a spread of
    # 0), so the bound is 10x that pair's spread plus 4 float32 ulps of the tensor's largest value.
    for n in names:
        d = float((getattr(c.model, n).detach() - final_a[n]).abs().max())
        spread = float((final_b[n] - final_a[n]).abs().max())
        ulps = 4 * torch.finfo(torch.float32).eps * float(final_a[n].abs().max())
        print(f"[{gs_type} resume] {n}: max |resumed - uninterrupted| {d:.3e}, run-to-run {spread:.3e}, 4 ulp {ulps:.3e}")
        assert d <= 10 * spread + ulps, (n, d, spread, ulps)
    # the saved iteration through cli.render and cli.metrics, each render at its view's size
    cli_render.main(["-m", out, "--gs_type", gs_type, "--skip_train", "--quiet"])
    for i, cam in enumerate(dataset.read_scene(root, "gs_flat", eval=True, shuffle=False).test_cameras):
        with open(os.path.join(out, "test", f"ours_{N_CLI}", f"renders_{gs_type}", f"{i:05d}.png"), "rb") as f:
            png = io_image.decode_png(f.read())
        assert png.shape[:2] == (cam.image_height, cam.image_width), i
    res = cli_metrics.main(["-m", out, "--gs_type", gs_type, "--quiet"])[out]
    for key in ("SSIM", "PSNR"):
        assert np.isfinite(res["results"][f"ours_{N_CLI}"][key])
