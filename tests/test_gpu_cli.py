"""The command-line programs end to end on the GPU (gms_b200.cli), on a small NeRF-synthetic scene rendered from a known
model: training of gs_mesh, gs_flat (densification and an opacity reset inside the run) and gs; the save timing against an
API loop that saves inside before_update; agreement with the API loop; resume; no host synchronisation in the loop; the
render and metrics programs against the library's renderers and the float64 metric restatement."""
import os

import numpy as np
import pytest
import torch

import metrics_restated
from gms_b200 import dataset, io_image, io_ply
from gms_b200.cli import metrics as cli_metrics
from gms_b200.cli import render as cli_render
from gms_b200.cli import train as cli_train
from gms_b200.model import FreeGaussianModel, MeshGaussianModel, PointsModel
from gms_b200.render import NativeFreeRenderer, NativeRenderer, PointsRenderer
from gms_b200.trainer import FreeTrainer, MeshTrainer
from test_gpu_dataset import _write_rendered_blender

pytestmark = pytest.mark.gpu

MESH_NAMES = ("vertices", "_alpha", "_scale", "_features", "_opacity")
MESH_ARGV = ["--eval", "--iterations", "30", "--test_iterations", "10", "--save_iterations", "10", "20",
             "--checkpoint_iterations", "15", "--quiet"]
FLAT_ARGV = ["--gs_type", "gs_flat", "--eval", "--iterations", "30", "--densify_from_iter", "5", "--densification_interval", "8",
             "--opacity_reset_interval", "20", "--densify_until_iter", "28", "--test_iterations", "-1", "--save_iterations", "12",
             "--checkpoint_iterations", "12", "--quiet"]
HOOKS_MESH, HOOKS_FLAT = {10, 20, 30}, {12, 30}     # report / save / last iterations of the two command lines


@pytest.fixture(scope="module")
def scene_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("cli_scene") / "scene")
    _write_rendered_blender(root)
    return root


def _params(model, names):
    return {n: getattr(model, n).detach().clone() for n in names}


def _within_spread(got, ref, other, what):
    """max |got - ref| <= 10 x max |other - ref| + 1e-7 per tensor, `other` a second run of the reference loop: the frames
    accumulate loss partial sums (and gs_mesh vertex gradients) with float atomics, so two runs of the same loop differ,
    and with densification the difference grows over the run (test_gpu_dataset.py's pattern)."""
    for n in ref:
        assert got[n].shape == ref[n].shape, f"{what}: {n} shapes {tuple(got[n].shape)} vs {tuple(ref[n].shape)}"
        d_got, d_other = float((got[n] - ref[n]).abs().max()), float((other[n] - ref[n]).abs().max())
        print(f"[{what}] {n}: max |got - ref| {d_got:.3e}, run-to-run {d_other:.3e}")
        assert d_got <= 10 * d_other + 1e-7, f"{what}: {n} {d_got:.3e} against the run-to-run {d_other:.3e}"


class _Recording(cli_train.Training):
    """Training that keeps a copy of the parameters it writes at every save."""

    def save(self, it):
        names = MESH_NAMES if self.args.gs_type == "gs_mesh" else FreeGaussianModel.NAMES
        self.saved = getattr(self, "saved", {})
        self.saved[it] = _params(self.model, names)
        super().save(it)


def _cli(root, out, argv, cls=cli_train.Training):
    return cls(cli_train.parse_args(["-s", root, "-m", out] + argv)).prepare().run()


def _api_mesh(root, out, iterations, hooks, saves):
    """The API loop: load_scene's view order, MeshTrainer, a before_update that saves at `saves`; returns (final parameters,
    parameters written at each save, parameters after each update that precedes a save)."""
    sc = dataset.load_scene(root, "gs_mesh", eval=True, num_splats=2)
    m = MeshGaussianModel.from_params(sc.mesh, "cuda", active_sh_degree=0, packed_features=True)
    tr = MeshTrainer(m, torch.zeros(3, device="cuda"), native=True)
    written, after = {}, {}
    for it, v in enumerate(sc.view_order(iterations), 1):
        def save(it=it):
            written[it] = os.path.join(out, f"iteration_{it}", "point_cloud.ply")
            io_ply.save_mesh_model(written[it], m)
        tr.optimizer_step = it < iterations
        hook = save if it in saves else (lambda: None)
        tr.step(sc.train_cameras[v], sc.train_images[v], before_update=hook if it in hooks else None)
        if it + 1 in saves:
            after[it] = _params(m, MESH_NAMES)
    return _params(m, MESH_NAMES), written, after


def _api_free(root, argv, hooks):
    args = cli_train.parse_args(["-s", root] + argv)
    sc = dataset.load_scene(root, args.gs_type, eval=True)
    m = FreeGaussianModel.from_point_cloud(*sc.point_cloud[:2], args.gs_type)
    tr = FreeTrainer(m, torch.zeros(3, device="cuda"), sc.cameras_extent, cli_train.free_params(args), white_background=False,
                     generator=torch.Generator(device="cuda").manual_seed(0))
    tr.losses = []
    for it, v in enumerate(sc.view_order(args.iterations), 1):
        tr.losses.append(tr.step(sc.train_cameras[v], sc.train_images[v], before_update=(lambda: None) if it in hooks else None).clone())
    tr.losses = torch.stack(tr.losses).tolist()
    return _params(m, FreeGaussianModel.NAMES), tr


@pytest.fixture(scope="module")
def mesh_run(scene_root, tmp_path_factory):
    out = str(tmp_path_factory.mktemp("cli_mesh"))
    return out, _cli(scene_root, out, MESH_ARGV, _Recording)


@pytest.fixture(scope="module")
def flat_run(scene_root, tmp_path_factory):
    out = str(tmp_path_factory.mktemp("cli_flat"))
    return out, _cli(scene_root, out, FLAT_ARGV, _Recording)


# ------------------------------------------------------------------------------------------------ train

def test_gs_mesh_trains_end_to_end(scene_root, mesh_run, tmp_path):
    out, run = mesh_run
    for f in ("cfg_args", "cameras.json", "input.ply", "chkpnt15.pth"):
        assert os.path.exists(os.path.join(out, f)), f
    assert [e for _, e in run.events] == [cli_train.iteration_events(it, run.args) for it in range(1, 31)]
    assert [it for it, _, _ in run.ema] == list(range(1, 31))
    ema = 0.0
    for it, loss, e in run.ema:
        ema = 0.4 * loss + 0.6 * ema
        assert e == ema and np.isfinite(loss)
    assert [(it, split) for it, split, _, _ in run.reports] == [(10, "test"), (10, "train")]
    for it in (10, 20, 30):
        p = io_ply.load_mesh_model(os.path.join(out, "point_cloud", f"iteration_{it}", "point_cloud.ply"))
        for n in ("vertices", "_alpha", "_scale", "_opacity"):
            assert torch.equal(getattr(p, n), run.saved[it][n].cpu()), f"iteration {it}: {n}"
        assert torch.equal(torch.cat((p._features_dc, p._features_rest), 1), run.saved[it]["_features"].cpu())
    # the API loop: what a save inside before_update writes is the parameters after N-1 updates, bit for bit
    final, written, after = _api_mesh(scene_root, str(tmp_path / "api"), 30, HOOKS_MESH, {10, 20, 30})
    for it in (10, 20, 30):
        p = io_ply.load_mesh_model(written[it])
        assert torch.equal(p._alpha, after[it - 1]["_alpha"].cpu()) and torch.equal(p._scale, after[it - 1]["_scale"].cpu())
        assert torch.equal(torch.cat((p._features_dc, p._features_rest), 1), after[it - 1]["_features"].cpu())
    assert not torch.equal(after[19]["_alpha"], after[29]["_alpha"])
    # agreement: the CLI against the API loop, within 10x the spread of two API runs
    final2, _, _ = _api_mesh(scene_root, str(tmp_path / "api2"), 30, HOOKS_MESH, set())
    _within_spread(_params(run.model, MESH_NAMES), final, final2, "gs_mesh CLI vs API")


def test_gs_mesh_resume_restores_state_bit_for_bit(scene_root, mesh_run, tmp_path):
    out, _ = mesh_run
    state, k = torch.load(os.path.join(out, "chkpnt15.pth"), map_location="cpu", weights_only=True)
    assert k == 15
    run = cli_train.Training(cli_train.parse_args(["-s", scene_root, "-m", str(tmp_path), "--start_checkpoint",
                                                   os.path.join(out, "chkpnt15.pth")] + MESH_ARGV)).prepare()
    now = run.trainer.state_dict()
    for key in ("p", "m", "v"):
        assert torch.equal(now["adam"][key].cpu(), state["trainer"]["adam"][key]), key
    assert now["adam"]["steps"] == state["trainer"]["adam"]["steps"] == [15] * len(now["adam"]["steps"])
    assert run.first_iter == 15 and run.order.state_dict() == state["view_order"]
    run.run()
    assert [it for it, _ in run.events] == list(range(16, 31))


def test_gs_mesh_loop_never_synchronises(scene_root, tmp_path):
    """Every iteration but the first, the report iterations and the save iterations runs under sync debug mode "error"."""
    sync_ok = {1, 10, 20, 30}

    class Strict(cli_train.Training):
        def _relaxed(self, fn, *a, **k):
            torch.cuda.set_sync_debug_mode(0)
            try:
                return fn(*a, **k)
            finally:
                torch.cuda.set_sync_debug_mode("error")

        def report(self, it):
            assert it in sync_ok
            self._relaxed(super().report, it)

        def save(self, it):
            assert it in sync_ok
            self._relaxed(super().save, it)

        def checkpoint(self, it):
            self._relaxed(super().checkpoint, it)

        def _consume(self, block=False):
            return self._relaxed(super()._consume, block) if block else super()._consume(block)

    run = Strict(cli_train.parse_args(["-s", scene_root, "-m", str(tmp_path)] + MESH_ARGV)).prepare()
    step = run.trainer.step

    def first_relaxed(*a, **k):
        return run._relaxed(step, *a, **k) if run._first else step(*a, **k)

    run._first = True
    run.trainer.step = lambda *a, **k: (first_relaxed(*a, **k), setattr(run, "_first", False))[0]
    torch.cuda.set_sync_debug_mode("error")
    try:
        run.run()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(run.ema) == 30


def test_gs_flat_trains_densifies_and_matches_api(scene_root, flat_run):
    out, run = flat_run
    tr = run.trainer
    assert [it for it, _, _ in tr.densifications] == [8, 16, 24]
    assert any("reset" in e for _, e in run.events)
    m = FreeGaussianModel.from_checkpoint(os.path.join(out, "point_cloud", "iteration_30", "point_cloud.ply"), "gs_flat")
    for n in FreeGaussianModel.NAMES:
        assert torch.equal(getattr(m, n).detach(), run.saved[30][n]), n
    m12 = FreeGaussianModel.from_checkpoint(os.path.join(out, "point_cloud", "iteration_12", "point_cloud.ply"), "gs_flat")
    assert m12.P == run.saved[12]["_xyz"].shape[0]
    a, ta = _api_free(scene_root, FLAT_ARGV, HOOKS_FLAT)
    b, tb = _api_free(scene_root, FLAT_ARGV, HOOKS_FLAT)
    print(f"[gs_flat] P: CLI {run.model.P}, API {ta.model.P} / {tb.model.P}; densifications CLI {tr.densifications}, "
          f"API {ta.densifications}; overflowed frames CLI {tr.frame.overflows}, API {ta.frame.overflows} / {tb.frame.overflows}")
    cli_losses = [l for _, l, _ in run.ema]
    first = lambda x, y: next((i + 1 for i, (p, q) in enumerate(zip(x, y)) if p != q), None)
    print(f"[gs_flat] first iteration whose loss differs: CLI vs API {first(cli_losses, ta.losses)}, API vs API {first(tb.losses, ta.losses)}")
    _within_spread(_params(run.model, FreeGaussianModel.NAMES), a, b, "gs_flat CLI vs API")


def test_gs_flat_resume_continues_the_run(scene_root, flat_run, tmp_path):
    out, full = flat_run
    ck = os.path.join(out, "chkpnt12.pth")
    state, k = torch.load(ck, map_location="cpu", weights_only=True)
    assert k == 12
    run = cli_train.Training(cli_train.parse_args(["-s", scene_root, "-m", str(tmp_path), "--start_checkpoint", ck] + FLAT_ARGV)).prepare()
    now = run.trainer.state_dict()
    for key in ("p", "m", "v"):
        assert torch.equal(now["adam"][key].cpu(), state["trainer"]["adam"][key]), key
    for key in ("accum", "denom", "generator"):
        assert torch.equal(now[key].cpu(), state["trainer"][key]), key
    assert now["adam"]["steps"] == state["trainer"]["adam"]["steps"] and now["P"] == state["trainer"]["P"] == run.model.P
    assert [it for it, _, _ in full.trainer.densifications if it < k] == [8]      # a densification before k ...
    run.run()
    assert [it for it, _, _ in run.trainer.densifications] == [16, 24]              # ... and two after it
    a, _ = _api_free(scene_root, FLAT_ARGV, HOOKS_FLAT)
    _within_spread(_params(run.model, FreeGaussianModel.NAMES), _params(full.model, FreeGaussianModel.NAMES), a,
                   "gs_flat resumed vs uninterrupted")


def test_gs_trains_end_to_end(scene_root, tmp_path):
    argv = ["--gs_type", "gs", "--eval", "--iterations", "20", "--densify_from_iter", "4", "--densification_interval", "6",
            "--test_iterations", "20", "--random_background", "--quiet"]
    run = _cli(scene_root, str(tmp_path), argv)
    assert [it for it, _, _ in run.trainer.densifications] == [6, 12, 18]
    m = FreeGaussianModel.from_checkpoint(str(tmp_path / "point_cloud" / "iteration_20" / "point_cloud.ply"), "gs")
    assert m.P == run.model.P and m.scale_cols == 3
    assert all(np.isfinite(l) for _, l, _ in run.ema) and len(run.reports) == 2


# ------------------------------------------------------------------------------------------------ render and metrics

def _expected_renders(model, renderer_cls, cams, bg, out_dir):
    r = renderer_cls(model, cams[0].image_width, cams[0].image_height)
    with io_image.ImageSink(cams[0].image_height, cams[0].image_width) as sink:
        for i, c in enumerate(cams):
            sink.write(r.render(c, bg)[0], os.path.join(out_dir, f"{i:05d}.png"))


@pytest.mark.parametrize("gs_type", ["gs_mesh", "gs_flat", "gs_points"])
def test_render_cli_matches_renderers(scene_root, mesh_run, flat_run, gs_type, tmp_path):
    out = (mesh_run if gs_type == "gs_mesh" else flat_run)[0]
    cli_render.main(["-m", out, "--gs_type", gs_type, "--quiet"])
    sc = dataset.load_scene(scene_root, "gs_flat", eval=True, shuffle=False)
    ply = os.path.join(out, "point_cloud", "iteration_30", "point_cloud.ply")
    model, cls = {"gs_mesh": lambda: (MeshGaussianModel.from_params(io_ply.load_mesh_model(ply), "cuda", packed_features=True), NativeRenderer),
                  "gs_flat": lambda: (FreeGaussianModel.from_checkpoint(ply, "gs_flat"), NativeFreeRenderer),
                  "gs_points": lambda: (PointsModel.from_flat_checkpoint(ply), PointsRenderer)}[gs_type]()
    bg = torch.zeros(3, device="cuda")
    for split, cams, images in (("train", sc.train_cameras, sc.train_images), ("test", sc.test_cameras, sc.test_images)):
        want = tmp_path / split
        _expected_renders(model, cls, cams, bg, str(want))
        got = os.path.join(out, split, "ours_30")
        for i in range(len(cams)):
            with open(os.path.join(got, f"renders_{gs_type}", f"{i:05d}.png"), "rb") as f, open(want / f"{i:05d}.png", "rb") as g:
                assert f.read() == g.read(), f"{split} {i}"
            with open(os.path.join(got, "gt", f"{i:05d}.png"), "rb") as f:
                assert np.array_equal(io_image.decode_png(f.read()), images[i].cpu().numpy()), f"{split} gt {i}"


def test_metrics_cli_matches_evaluate_and_restatement(scene_root, flat_run):
    out = flat_run[0]
    cli_render.main(["-m", out, "--gs_type", "gs_flat", "--skip_train", "--quiet"])
    res = cli_metrics.main(["-m", out, "--gs_type", "gs_flat", "--quiet"])[out]
    pv = res["per_view"]["ours_30"]
    sc = dataset.load_scene(scene_root, "gs_flat", eval=True, shuffle=False)
    model = FreeGaussianModel.from_checkpoint(os.path.join(out, "point_cloud", "iteration_30", "point_cloud.ply"), "gs_flat")
    r = NativeFreeRenderer(model, sc.test_cameras[0].image_width, sc.test_cameras[0].image_height)
    ev = r.evaluate(sc.test_cameras, sc.test_images, torch.zeros(3, device="cuda"), protocol="metrics").per_view
    worst = [0.0, 0.0]
    for name in pv["SSIM"]:
        i = int(name[:5])
        for key, col in (("SSIM", 1), ("PSNR", 2)):
            worst[col - 1] = max(worst[col - 1], abs(pv[key][name] - float(np.float32(ev[i, col]))))
        d = os.path.join(out, "test", "ours_30")
        with open(os.path.join(d, "renders_gs_flat", name), "rb") as f, open(os.path.join(d, "gt", name), "rb") as g:
            x = torch.from_numpy(io_image.decode_png(f.read())).permute(2, 0, 1).float() / 255.0
            y = torch.from_numpy(io_image.decode_png(g.read())).permute(2, 0, 1).float() / 255.0
        ref = metrics_restated.metrics64(x, y, "training_report")
        assert abs(pv["SSIM"][name] - ref[1]) <= 2e-6 and abs(pv["PSNR"][name] - ref[2]) <= 1e-4, name
    print(f"[metrics CLI vs evaluate(metrics)] largest difference: SSIM {worst[0]:.3e}, PSNR {worst[1]:.3e} dB")
    assert worst == [0.0, 0.0]
    assert os.path.exists(os.path.join(out, "results_gs_flat.json")) and os.path.exists(os.path.join(out, "per_view_gs_flat.json"))
