"""The cost of cli.train's TensorBoard logging: the command-line loop with TensorBoard against the same loop with
torch.utils.tensorboard hidden from the import (what the program does when TensorBoard is not installed), on
tools/train_cli_eval.py's generated 1080p NeRF-synthetic scene.

    python tools/train_cli_tb_eval.py --out DIR                 # writes the scene
    python tools/train_cli_tb_eval.py --out DIR --bench         # ... and measures

Workloads: gs_mesh at 1M mesh-Gaussians (--num_splats 5), and gs_flat from the random 100k cloud with densification every
50 iterations.  Reports and saves are off, so the difference is the one event per iteration with its three scalars, the
timing events and the writer's thread.  A third arm, "per_tag", writes the three scalars with one add_scalar each (one
event per tag, as the reference does), to show what the single event saves.  `--runs` alternating runs per arm, each a
host clock around `--steps` iterations ending in a device synchronisation (the scene is loaded once, outside the clock);
medians.  Also printed: the host time of one per-iteration event and of three add_scalar calls into a scratch writer.
The card's name and power limit are printed in the same run."""
import argparse
import contextlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import train_cli_eval as tce  # noqa: E402  (puts the package and tests/ on sys.path)
import numpy as np  # noqa: E402

from gms_b200 import dataset  # noqa: E402
from gms_b200.cli import train as cli_train  # noqa: E402


def bench(root, out, gs_type, steps, runs, extra):
    argv = ["-s", root, "-m", os.path.join(out, f"tb_{gs_type}"), "--gs_type", gs_type, "--eval", "--iterations", str(steps),
            "--test_iterations", "-1", "--quiet"] + extra
    if gs_type == "gs_mesh":
        argv += ["--num_splats", "5"]
    args = cli_train.parse_args(argv)
    scene = dataset.load_scene(root, gs_type, eval=True, num_splats=args.num_splats[0])

    def arm(tensorboard, per_tag=False):
        with contextlib.nullcontext() if tensorboard else tce.tensorboard_hidden():
            t = (_PerTag if per_tag else tce._NoSave)(cli_train.parse_args(argv), scene=scene).prepare()
        assert (t.tb_writer is not None) == tensorboard
        dt, _ = tce._timed(t.run)
        return dt, len(getattr(t.trainer, "densifications", []))

    arm(True), arm(False)      # warm-up
    res = {"tensorboard": [], "hidden": [], "per_tag": [], "densifications": None}
    for _ in range(runs):
        for name, tb in (("tensorboard", True), ("hidden", False), ("per_tag", True)):
            dt, nd = arm(tb, per_tag=name == "per_tag")
            res[name].append(1e3 * dt / steps)
            res["densifications"] = nd
    a, b, u = (float(np.median(res[k])) for k in ("tensorboard", "hidden", "per_tag"))
    res.update(tensorboard_median_ms=a, hidden_median_ms=b, per_tag_median_ms=u, diff_ms=a - b, diff_pct=100 * (a - b) / b,
               per_tag_diff_ms=u - b, per_tag_diff_pct=100 * (u - b) / b)
    print(json.dumps({gs_type: res}), flush=True)
    return res


class _PerTag(tce._NoSave):
    def log_iteration(self, it, loss, l1, ms):
        w = self.tb_writer
        w.add_scalar("train_loss_patches/l1_loss", l1, it)
        w.add_scalar("train_loss_patches/total_loss", loss, it)
        w.add_scalar("iter_time", ms, it)


def event_cost(out, n=3000):
    """Host microseconds per iteration's scalars into a scratch writer, the writer's thread included (closed inside the
    clock): Training.log_iteration (one event) and the three add_scalar calls of the per_tag arm."""
    import time
    from torch.utils.tensorboard import SummaryWriter
    res = {}
    for name, cls in (("one_event_us", cli_train.Training), ("per_tag_us", _PerTag)):
        t = cls(cli_train.parse_args(["-s", out, "-m", out, "--quiet"]), device="cpu")
        t.tb_writer = SummaryWriter(os.path.join(out, f"event_cost_{name}"))
        t0 = time.perf_counter()
        for i in range(n):
            t.log_iteration(i, 0.1, 0.05, 2.1)
        t.close_writer()
        res[name] = 1e6 * (time.perf_counter() - t0) / n
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--faces", type=int, default=200_000)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    root = os.path.join(a.out, "scene")
    if not os.path.exists(os.path.join(root, "transforms_train.json")):
        dt, _ = tce._timed(lambda: tce.write_scene(root, a.views, a.faces))
        print(f"scene written in {dt:.1f} s", flush=True)
    if not a.bench:
        return
    print(tce.card(), flush=True)
    event_cost(a.out)
    bench(root, a.out, "gs_mesh", a.steps, a.runs, [])
    bench(root, a.out, "gs_flat", a.steps, a.runs, ["--densify_from_iter", "50", "--densification_interval", "50"])
    print(tce.card(), flush=True)


if __name__ == "__main__":
    main()
