"""The command-line programs (gms_b200.cli) against bare API loops, on a generated 1080p NeRF-synthetic scene.

    python tools/train_cli_eval.py --out DIR                 # writes the scene
    python tools/train_cli_eval.py --out DIR --bench         # ... and measures

Scene (deterministic): `--views` views at 1920x1080 (the last fifth held out as test views) rendered by the native renderer
from a seeded scenes.object_mesh(200_000) gs_mesh model, written as RGBA PNGs (alpha 255) with transforms_*.json, plus the
mesh as mesh.obj: 1M mesh-Gaussians at --num_splats 5.
Measurements, `--runs` alternating runs per arm, each a host clock around `--steps` iterations ending in a device
synchronisation (the scene is loaded once, outside the clock):
  gs_mesh   cli.train's loop (reports and saves off, TensorBoard hidden from the import: its cost is
            tools/train_cli_tb_eval.py's to measure) against a bare MeshTrainer.step loop over the same view order
  gs_flat   the same with densification on (from the random 100k cloud), FreeTrainer.step as the bare loop; the number of
            densification steps inside the window is printed beside the times
  render    cli.render over the test views: views per second (PNGs written)
  metrics   cli.metrics over the rendered test views: seconds
The card's name and power limit are printed in the same run."""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gms_b200 import dataset, io_image, scenes  # noqa: E402
from gms_b200.cli import metrics as cli_metrics  # noqa: E402
from gms_b200.cli import render as cli_render  # noqa: E402
from gms_b200.cli import train as cli_train  # noqa: E402
from gms_b200.model import FreeGaussianModel, MeshGaussianModel  # noqa: E402
from gms_b200.render import NativeRenderer  # noqa: E402
from gms_b200.trainer import FreeTrainer, MeshTrainer  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable: {e}"


def write_scene(root, views, faces, W=1920, H=1080):
    import dataset_cases
    verts, fcs = scenes.object_mesh(faces)
    model = MeshGaussianModel.from_params(scenes.init_mesh_gaussians(verts, fcs, K=1, seed=3), "cuda", packed_features=True)
    r = NativeRenderer(model, W, H)
    ring = scenes.ring_cameras(views, 3.2, W, H, elevation_deg=20.0)
    n_test = max(1, views // 5)
    bg = torch.zeros(3, device="cuda")
    for split, cams in (("train", ring[:views - n_test]), ("test", ring[views - n_test:])):
        os.makedirs(os.path.join(root, split), exist_ok=True)
        frames = []
        for i, c in enumerate(cams):
            rgb = io_image.quantize(r.render(c.to("cuda"), bg)[0]).cpu().numpy().reshape(H, W, 3)
            dataset_cases.write_png(os.path.join(root, split, f"r_{i}.png"), np.concatenate([rgb, np.full((H, W, 1), 255, np.uint8)], 2))
            c2w = np.linalg.inv(c.world_view_transform.numpy().T.astype(np.float64))
            c2w[:3, 1:3] *= -1
            frames.append({"file_path": f"./{split}/r_{i}", "transform_matrix": c2w.tolist()})
        with open(os.path.join(root, f"transforms_{split}.json"), "w") as f:
            json.dump({"camera_angle_x": scenes.NERF_FOVX, "frames": frames}, f)
    # the loader applies transform_vertices (y <-> z, new y negated): store the inverse so the trained mesh is the rendered one
    v = np.stack([verts[:, 0], verts[:, 2], -verts[:, 1]], 1)
    with open(os.path.join(root, "mesh.obj"), "w") as f:
        f.write("".join("v %.6f %.6f %.6f\n" % tuple(x) for x in v))
        f.write("".join("f %d %d %d\n" % tuple(t) for t in fcs + 1))


@contextlib.contextmanager
def tensorboard_hidden():
    """torch.utils.tensorboard fails to import inside the block, as when TensorBoard is not installed: a Training prepared
    there writes no event file."""
    saved = sys.modules.get("torch.utils.tensorboard")
    sys.modules["torch.utils.tensorboard"] = None
    try:
        yield
    finally:
        if saved is not None:
            sys.modules["torch.utils.tensorboard"] = saved
        else:
            sys.modules.pop("torch.utils.tensorboard", None)


class _NoSave(cli_train.Training):
    def save(self, it):
        pass


def _timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t), out


def bench_train(root, out, gs_type, steps, runs, extra):
    argv = ["-s", root, "-m", os.path.join(out, f"run_{gs_type}"), "--gs_type", gs_type, "--eval", "--iterations", str(steps),
            "--test_iterations", "-1", "--quiet"] + extra
    if gs_type == "gs_mesh":
        argv += ["--num_splats", "5"]
    args = cli_train.parse_args(argv)
    scene = dataset.load_scene(root, gs_type, eval=True, num_splats=args.num_splats[0])
    order = scene.view_order(steps)

    def cli():
        with tensorboard_hidden():
            t = _NoSave(cli_train.parse_args(argv), scene=scene).prepare()
        dt, _ = _timed(t.run)
        return dt, len(getattr(t.trainer, "densifications", []))

    def bare():
        bg = torch.zeros(3, device="cuda")
        if gs_type == "gs_mesh":
            m = MeshGaussianModel.from_params(scene.mesh, "cuda", active_sh_degree=0, packed_features=True)
            tr = MeshTrainer(m, bg, native=True)
        else:
            m = FreeGaussianModel.from_point_cloud(*scene.point_cloud[:2], gs_type)
            tr = FreeTrainer(m, bg, scene.cameras_extent, cli_train.free_params(args),
                             generator=torch.Generator(device="cuda").manual_seed(0))

        def loop():
            for i, v in enumerate(order):
                if gs_type == "gs_mesh":
                    tr.optimizer_step = i + 1 < steps
                tr.step(scene.train_cameras[v], scene.train_images[v])
        dt, _ = _timed(loop)
        return dt, len(getattr(tr, "densifications", []))

    cli(), bare()       # warm-up
    res = {"cli": [], "bare": [], "densifications": None}
    for _ in range(runs):
        for name, fn in (("cli", cli), ("bare", bare)):
            dt, nd = fn()
            res[name].append(1e3 * dt / steps)
            res["densifications"] = nd
    c, b = float(np.median(res["cli"])), float(np.median(res["bare"]))
    res.update(cli_median_ms=c, bare_median_ms=b, diff_ms=c - b, diff_pct=100 * (c - b) / b, P=None)
    print(json.dumps({gs_type: res}), flush=True)
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
        dt, _ = _timed(lambda: write_scene(root, a.views, a.faces))
        print(f"scene written in {dt:.1f} s", flush=True)
    if not a.bench:
        return
    print(card(), flush=True)
    bench_train(root, a.out, "gs_mesh", a.steps, a.runs, [])
    bench_train(root, a.out, "gs_flat", a.steps, a.runs, ["--densify_from_iter", "50", "--densification_interval", "50"])
    # render and metrics over the gs_mesh run's model: one full run with its save
    model_dir = os.path.join(a.out, "run_gs_mesh")
    cli_train.main(["-s", root, "-m", model_dir, "--eval", "--iterations", "10", "--test_iterations", "-1", "--num_splats", "5",
                    "--quiet"])
    n = None
    for k in range(2):
        dt, r = _timed(lambda: cli_render.main(["-m", model_dir, "--gs_type", "gs_mesh", "--skip_train", "--quiet"]))
        n = r["views"]["test"]
        print(json.dumps({"render": {"views": n, "seconds": dt, "views_per_s": n / dt, "warm": k == 1}}), flush=True)
    for k in range(2):
        dt, _ = _timed(lambda: cli_metrics.main(["-m", model_dir, "--gs_type", "gs_mesh", "--quiet"]))
        print(json.dumps({"metrics": {"views": n, "seconds": dt, "warm": k == 1}}), flush=True)


if __name__ == "__main__":
    main()
