"""cli.train's TensorBoard event files on the GPU, read back with TensorBoard's event loader: gs_mesh and gs_flat (with
densifications inside the run) at test_gpu_cli.py's sizes, gs_multi_mesh and gs_flame on test_gpu_train_mesh_types.py's
scenes.  Per iteration: total_loss is the loss the progress display consumed, l1_loss element 1 of the frame's device loss
vector, iter_time one finite positive value.  At report iterations: the renders of the first five views of each split
against a native render of the checkpoint saved at that iteration, the ground truth at the first listed test iteration
only, the split scalars, the opacity histogram and total_points.  Also: no host synchronisation in a TensorBoard-enabled
loop, a second event file on resume, and no event file with torch.utils.tensorboard hidden."""
import os
import shutil
import sys

import numpy as np
import pytest
import torch

pytest.importorskip("tensorboard")

import mesh_types_cases as cases  # noqa: E402
import tensorboard_events as tbe  # noqa: E402
from gms_b200.cli import render as cli_render  # noqa: E402
from gms_b200.cli import train as cli_train  # noqa: E402
from test_gpu_dataset import _write_rendered_blender  # noqa: E402
from test_gpu_train_mesh_types import _write_colmap_from_blender  # noqa: E402

pytestmark = pytest.mark.gpu

N = 30
COMMON = ["--eval", "--iterations", str(N), "--test_iterations", "10", "20", "--save_iterations", "10", "20",
          "--checkpoint_iterations", "15", "--quiet"]
ARGV = {
    "gs_mesh": COMMON,
    # densifications at 8, 16 and 24 with a zero gradient threshold (every Gaussian is cloned or split): P differs between
    # the reports at 12 and 24
    "gs_flat": ["--gs_type", "gs_flat", "--eval", "--iterations", str(N), "--densify_from_iter", "5", "--densification_interval", "8",
                "--densify_grad_threshold", "0", "--opacity_reset_interval", "20", "--densify_until_iter", "28", "--test_iterations", "12", "24",
                "--save_iterations", "12", "24", "--quiet"],
    "gs_multi_mesh": ["--gs_type", "gs_multi_mesh", "--meshes", "a", "b", "--num_splats", "2", "3"] + COMMON,
    "gs_flame": ["--gs_type", "gs_flame", "--flame_model", cases.FLAME_MODEL] + COMMON,
}


@pytest.fixture(scope="module")
def roots(tmp_path_factory):
    base = tmp_path_factory.mktemp("tb_scenes")
    blender = str(base / "blender")
    _write_rendered_blender(blender)
    return {"blender": blender, "colmap": _write_colmap_from_blender(blender, str(base / "colmap"))}


def _root(roots, gs_type):
    return roots["colmap" if gs_type == "gs_multi_mesh" else "blender"]


class _Vectors(cli_train.Training):
    """Training that keeps a device copy of every frame's [loss, L1, SSIM] vector (stream-ordered, no synchronisation)."""

    def _setup(self):
        super()._setup()
        step, self.vectors = self.trainer.step, []

        def recorded(*a, **k):
            out = step(*a, **k)
            tr = self.trainer
            self.vectors.append((tr._frame.loss if isinstance(tr, cli_train.MeshTrainer) else tr.loss_vector).clone())
            return out
        self.trainer.step = recorded
        return self


@pytest.fixture(scope="module")
def runs(roots, tmp_path_factory):
    return {}


def _run(runs, roots, tmp_path_factory, gs_type):
    if gs_type not in runs:
        out = str(tmp_path_factory.mktemp(f"tb_{gs_type}"))
        run = _Vectors(cli_train.parse_args(["-s", _root(roots, gs_type), "-m", out] + ARGV[gs_type])).prepare().run()
        runs[gs_type] = (out, run)
    return runs[gs_type]


def _checkpoint_render(out, gs_type, it, cam, bg):
    """trunc(clamp(render, 0, 1) * 255) of point_cloud/iteration_<it> drawn by the native renderer, at SH degree 0 (the
    degree of every iteration below 1000), and the checkpoint's model."""
    ply = os.path.join(out, "point_cloud", f"iteration_{it}", "point_cloud.ply")
    model, cls = cli_render.load_model(gs_type, ply, 3, torch.device("cuda"))
    model.active_sh_degree = 0
    img = cls(model, cam.image_width, cam.image_height).render(cam, bg)[0]
    png = (torch.clamp(img, 0.0, 1.0).permute(1, 2, 0).cpu().numpy() * np.float32(255)).astype(np.uint8)
    return png, model


@pytest.mark.parametrize("gs_type", ["gs_mesh", "gs_flat", "gs_multi_mesh", "gs_flame"])
def test_event_file_holds_training_report(runs, roots, tmp_path_factory, gs_type):
    out, run = _run(runs, roots, tmp_path_factory, gs_type)
    files = tbe.event_files(out)
    assert len(files) == 1 and run.tb_writer is not None
    tags = tbe.read_events(files[0])
    for tag, ev in tags.items():
        steps = [s for s, _ in ev]
        assert steps == sorted(steps), tag
    # per iteration
    vec = torch.stack(run.vectors).cpu().numpy()
    assert vec.shape == (N, 3)
    want_total = [(it, float(np.float32(loss))) for it, loss, _ in run.ema]
    assert [it for it, _ in want_total] == list(range(1, N + 1))
    assert tags["train_loss_patches/total_loss"] == want_total
    assert tags["train_loss_patches/l1_loss"] == [(it, float(vec[it - 1, 1])) for it in range(1, N + 1)]
    assert np.array_equal(vec[:, 0], np.array([l for _, l, _ in run.ema], dtype=np.float32))
    times = tags["iter_time"]
    assert [s for s, _ in times] == list(range(1, N + 1)) and all(np.isfinite(t) and t > 0 for _, t in times)
    print(f"[{gs_type}] iter_time median {np.median([t for _, t in times]):.3f} ms")
    # report iterations
    reports = run.args.test_iterations
    bg = torch.zeros(3, device="cuda")
    worst = 0
    for it in reports:
        P = None
        for name, cams, gts, names in cli_train.report_configs(run.scene):
            for k, (cam, gt, image_name) in enumerate(zip(cams, gts, names)):
                tag = f"{name}_view_{image_name}"
                if k >= 5:
                    assert all(s != it for s, _ in tags.get(tag + "/render", [])), tag
                    continue
                want, model = _checkpoint_render(out, gs_type, it, cam, bg)
                P = int(model._opacity.shape[0])
                repeats = names[:5].count(image_name)       # a view the train config's mod n repeats is logged each time
                got = [png for s, png in tags[tag + "/render"] if s == it]
                assert len(got) == repeats, tag
                d = max(int(np.abs(g.astype(np.int32) - want.astype(np.int32)).max()) for g in got)
                worst = max(worst, d)
                if gs_type == "gs_flame":       # the checkpoint's pose comes from the FLAME model rebuilt from the file
                    assert d <= 1, f"{tag} at {it}: {d}"
                else:
                    assert d == 0, f"{tag} at {it}: {d}"
                gt_events = [png for s, png in tags.get(tag + "/ground_truth", []) if s == it]
                if it == reports[0]:
                    b = gt.cpu().numpy()
                    want_gt = ((b / np.float32(255)).astype(np.float32) * np.float32(255)).astype(np.uint8)
                    assert len(gt_events) == repeats and all(np.array_equal(g, want_gt) for g in gt_events), tag
                else:
                    assert gt_events == [], tag
            rep = [(l1, psnr) for i, s, l1, psnr in run.reports if i == it and s == name]
            if cams:
                assert [v for s, v in tags[f"{name}/loss_viewpoint - l1_loss"] if s == it] == [float(np.float32(rep[0][0]))]
                assert [v for s, v in tags[f"{name}/loss_viewpoint - psnr"] if s == it] == [float(np.float32(rep[0][1]))]
        _, model = _checkpoint_render(out, gs_type, it, run.scene.test_cameras[0], bg)
        op = torch.sigmoid(model._opacity.detach()).cpu().numpy()
        [h] = [h for s, h in tags["scene/opacity_histogram"] if s == it]
        assert h.num == op.size == P and h.min == float(op.min()) and h.max == float(op.max())
        assert [v for s, v in tags["total_points"] if s == it] == [float(P)]
    print(f"[{gs_type}] largest render PNG difference against the checkpoint's render: {worst}")
    if gs_type == "gs_flat":
        assert [it for it, _, _ in run.trainer.densifications] == [8, 16, 24]
        points = [v for _, v in tags["total_points"]]
        print(f"[gs_flat] total_points at 12 and 24: {points}")
        assert points[0] != points[1]


def test_loop_with_tensorboard_never_synchronises(roots, tmp_path):
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

    run = Strict(cli_train.parse_args(["-s", roots["blender"], "-m", str(tmp_path)] + ARGV["gs_mesh"])).prepare()
    assert run.tb_writer is not None
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
    assert len(run.ema) == N
    tags = tbe.read_events(tbe.event_files(str(tmp_path))[0])
    assert [s for s, _ in tags["iter_time"]] == list(range(1, N + 1))


def test_resume_writes_a_second_event_file(runs, roots, tmp_path_factory, tmp_path):
    out, _ = _run(runs, roots, tmp_path_factory, "gs_mesh")
    resumed = str(tmp_path / "model")
    shutil.copytree(out, resumed)
    first = tbe.event_files(resumed)
    run = cli_train.Training(cli_train.parse_args(["-s", roots["blender"], "-m", resumed, "--start_checkpoint",
                                                   os.path.join(resumed, "chkpnt15.pth")] + COMMON)).prepare().run()
    files = tbe.event_files(resumed)
    assert len(first) == 1 and len(files) == 2 and files[0] == first[0]
    tags = tbe.read_events(files[1])
    for tag in ("train_loss_patches/total_loss", "train_loss_patches/l1_loss", "iter_time"):
        assert [s for s, _ in tags[tag]] == list(range(16, N + 1)), tag
    assert tags["train_loss_patches/total_loss"] == [(it, float(np.float32(l))) for it, l, _ in run.ema]
    assert [s for s, _ in tags["total_points"]] == [20]          # the report at 10 is before the checkpoint
    assert not any(t.endswith("/ground_truth") for t in tags)       # 20 is not the first listed test iteration


def test_hidden_tensorboard_writes_no_event_file(roots, tmp_path, monkeypatch):
    monkeypatch.setitem(sys.modules, "torch.utils.tensorboard", None)
    argv = ["--eval", "--iterations", "5", "--test_iterations", "5", "--quiet"]
    run = cli_train.Training(cli_train.parse_args(["-s", roots["blender"], "-m", str(tmp_path)] + argv)).prepare().run()
    assert run.tb_writer is None and len(run.ema) == 5 and len(run.reports) == 2
    assert not [f for f in os.listdir(tmp_path) if f.startswith("events.out.tfevents.")]
