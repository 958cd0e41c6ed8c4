"""cli.train's TensorBoard logging on the host: Training.report and Training.log_iteration, with a recording writer, make the
calls the reference's own training_report makes (tests/golden/tensorboard.npz, written by make_tensorboard_golden.py), tag
by tag; through a real SummaryWriter the stored PNGs are TensorBoard's truncation of those floats; the writer's lifecycle;
and with torch.utils.tensorboard hidden, the reference's message and no event file."""
import os
import sys
from argparse import Namespace
from collections import defaultdict
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from gms_b200.cli import train as cli_train

CASES = ("outside", "first", "later", "empty_test", "few_test", "first_unreached")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "tensorboard.npz"))


class Recorder:
    """SummaryWriter's calls as (method, tag, step, value); a summary handed to file_writer.add_summary is recorded as one
    add_scalar per simple_value (float32, as the event file stores it)."""

    def __init__(self):
        self.calls = []
        self.file_writer = self

    def add_summary(self, summary, global_step=None):
        for v in summary.value:
            self.calls.append(("add_scalar", v.tag, global_step, float(v.simple_value)))

    def add_scalar(self, tag, value, global_step=None):
        self.calls.append(("add_scalar", tag, global_step, float(value)))

    def add_images(self, tag, img, global_step=None):
        self.calls.append(("add_images", tag, global_step, np.array(img.numpy(), dtype=np.float32)))

    def add_histogram(self, tag, values, global_step=None):
        self.calls.append(("add_histogram", tag, global_step, np.array(values.numpy(), dtype=np.float32)))


class _Renderer:
    def render(self, cam, bg):
        return cam.image.clone(), None, None


class _Trainer:
    """evaluate(): training_report's float64 means of the per-view L1 and PSNR (columns 0 and 3), and a renderer.  This
    stand-in computes the split metrics itself, so the loss_viewpoint comparison below pins the tags, the steps and that
    Training passes evaluate()'s means through; that the native evaluate() computes them right is
    test_gpu_tensorboard.py's check against the run's reports (and test_gpu_cli.py's)."""
    bg = torch.zeros(3)
    renderer = None

    def evaluate(self, cams, gts):
        self.renderer = _Renderer()
        l1 = psnr = 0.0
        for c, g in zip(cams, gts):
            x, y = torch.clamp(c.image, 0.0, 1.0), g.permute(2, 0, 1) / 255.0
            l1 += float(torch.abs(x - y).mean().double())
            mse = ((x - y) ** 2).view(3, -1).mean(1)
            psnr += float((20 * torch.log10(1.0 / torch.sqrt(mse))).mean().double())
        return SimpleNamespace(mean=torch.tensor([l1 / len(cams), 0.0, 0.0, psnr / len(cams)], dtype=torch.float64))


def native_run(g, case, writer):
    """Training's TensorBoard calls for one golden case, on a scene of stand-in cameras that carry the case's renders."""
    split = {}
    for s in ("train", "test"):
        renders, gts = g[f"{case}/{s}/renders"], g[f"{case}/{s}/gt"]
        split[s] = ([SimpleNamespace(image=torch.from_numpy(r)) for r in renders], [torch.from_numpy(x) for x in gts],
                    [str(n) for n in g[f"{case}/{s}/names"]])
    scene = SimpleNamespace(train_cameras=split["train"][0], train_images=split["train"][1], train_names=split["train"][2],
                            test_cameras=split["test"][0], test_images=split["test"][1], test_names=split["test"][2])
    it, tests = int(g[f"{case}/iteration"]), [int(x) for x in g[f"{case}/test_iterations"]]
    t = cli_train.Training(Namespace(quiet=True, test_iterations=tests), device="cpu", scene=scene)
    t.trainer, t.model = _Trainer(), SimpleNamespace(get_opacity=torch.sigmoid(torch.from_numpy(g[f"{case}/opacity_logits"])))
    t.tb_writer = writer
    t.log_iteration(it, float(g[f"{case}/loss"]), float(g[f"{case}/l1"]), float(g[f"{case}/elapsed"]))
    if it in tests:
        t.report(it)
    return t


def golden_calls(g, case):
    calls, k = [], 0
    while f"{case}/call/{k}/method" in g:
        p = f"{case}/call/{k}/"
        calls.append((str(g[p + "method"]), str(g[p + "tag"]), int(g[p + "step"]), g[p + "value"]))
        k += 1
    return calls


def by_tag(calls):
    out = defaultdict(list)
    for method, tag, step, value in calls:
        out[tag].append((method, step, value))
    return out


@pytest.mark.parametrize("case", CASES)
def test_report_and_scalars_make_the_reference_calls(golden, case):
    want = by_tag(golden_calls(golden, case))
    got = by_tag(native_run(golden, case, Recorder()).tb_writer.calls)
    assert sorted(got) == sorted(want)
    for tag in want:
        assert [(m, s) for m, s, _ in got[tag]] == [(m, s) for m, s, _ in want[tag]], tag
        for (m, _, a), (_, _, b) in zip(got[tag], want[tag]):
            if m == "add_scalar" and "loss_viewpoint" in tag:      # float64 means: the sum's order may differ in the last bits
                assert a == pytest.approx(float(b), rel=1e-12, abs=1e-15), tag
            elif m == "add_scalar":     # per-iteration values: float32 in the event, as add_scalar's simple_value
                assert np.float32(a) == np.float32(b), tag
            else:
                assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), tag
    if case == "first":
        assert any(t.endswith("/ground_truth") for t in want)
    if case in ("later", "first_unreached"):
        assert not any(t.endswith("/ground_truth") for t in want)


def test_stored_pngs_are_tensorboards_truncation(golden, tmp_path):
    """Through SummaryWriter: each render PNG is trunc(clamp(render, 0, 1) * 255) and each ground truth PNG
    trunc(float32(b / 255) * 255)."""
    pytest.importorskip("tensorboard")
    from torch.utils.tensorboard import SummaryWriter
    import tensorboard_events as tbe
    g, case = golden, "first"
    w = SummaryWriter(str(tmp_path))
    native_run(g, case, w)
    w.close()
    files = tbe.event_files(str(tmp_path))
    assert len(files) == 1
    tags = tbe.read_events(files[0])
    n_test = len(g[f"{case}/test/names"])
    for i, name in enumerate(g[f"{case}/test/names"][:5]):
        [(step, png)] = tags[f"test_view_{name}/render"]
        x = np.clip(g[f"{case}/test/renders"][i], 0, 1).transpose(1, 2, 0)
        assert step == 7 and np.array_equal(png, (x * np.float32(255)).astype(np.uint8))
        [(_, gt_png)] = tags[f"test_view_{name}/ground_truth"]
        b = g[f"{case}/test/gt"][i]
        assert np.array_equal(gt_png, ((b / np.float32(255)).astype(np.float32) * np.float32(255)).astype(np.uint8))
    assert n_test > 5 and f"test_view_{g[f'{case}/test/names'][5]}/render" not in tags
    [(_, h)] = tags["scene/opacity_histogram"]
    op = 1 / (1 + np.exp(-g[f"{case}/opacity_logits"].astype(np.float64)))
    assert h.num == op.size and h.min == pytest.approx(op.min(), rel=1e-6) and h.max == pytest.approx(op.max(), rel=1e-6)
    assert tags["total_points"] == [(7, float(op.size))]
    assert tags["train_loss_patches/total_loss"] == [(7, float(g[f"{case}/loss"]))]


class _OutputOnly(cli_train.Training):
    """prepare() up to the output directory and the writer."""

    def _setup(self):
        return self


def _args(tmp_path, quiet=False):
    return cli_train.parse_args(["-s", str(tmp_path / "missing_scene"), "-m", str(tmp_path / "out")] + (["--quiet"] if quiet else []))


def test_without_tensorboard_prints_the_message_and_writes_no_event_file(tmp_path, monkeypatch, capsys):
    monkeypatch.setitem(sys.modules, "torch.utils.tensorboard", None)      # import fails as when tensorboard is absent
    t = _OutputOnly(_args(tmp_path)).prepare()
    assert t.tb_writer is None
    assert "Tensorboard not available: not logging progress" in capsys.readouterr().out.splitlines()
    assert sorted(os.listdir(tmp_path / "out")) == ["cfg_args"]


def test_writer_opens_in_prepare_and_closes_when_setup_fails(tmp_path):
    pytest.importorskip("tensorboard")

    class Failing(cli_train.Training):
        def _setup(self):
            self.seen = self.tb_writer
            raise RuntimeError("scene")

    t = Failing(_args(tmp_path, quiet=True))
    with pytest.raises(RuntimeError, match="scene"):
        t.prepare()
    assert t.seen is not None
    files = [f for f in os.listdir(tmp_path / "out") if f.startswith("events.out.tfevents.")]
    assert len(files) == 1
    assert t.tb_writer.all_writers is None          # SummaryWriter.close() drops its file writers
