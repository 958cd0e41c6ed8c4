"""cli.render_time_animated against a bare API loop over the same frames, on a generated 1080p NeRF-synthetic scene.

    python tools/scripts_cli_eval.py --out DIR --bench

Scene: train_cli_eval.write_scene (`--views` views at 1920x1080, the last fifth held out as test views, rendered from a
seeded scenes.object_mesh(200_000) model), and a gs_mesh checkpoint of that mesh at --num_splats 5 (1M mesh-Gaussians,
seeded parameters) with its cfg_args.  Measured, `--runs` alternating runs per arm over the train views, each a host clock
ending in a device synchronisation after every PNG is written:
  program  cli.render_time_animated's frame loop (render.render_frames: transform_hotdog_fly, NativeRenderer.render(
           vertices=...), ImageSink.write; the ground-truth PNGs are not written in these runs, the scene and checkpoint
           are loaded outside the clock)
  bare     the same frames through NativeRenderer.render(vertices=...) and ImageSink.write in a plain loop
Frames per second of each, and the program's overhead.  The card's name and power limit are printed in the same run."""
import argparse
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import torch  # noqa: E402

import train_cli_eval  # noqa: E402
from gms_b200 import io_image, io_ply, scenes  # noqa: E402
from gms_b200.cli import render as cli_render  # noqa: E402
from gms_b200.cli import render_time_animated  # noqa: E402
from gms_b200.model import MeshGaussianModel  # noqa: E402
from gms_b200.render import NativeRenderer  # noqa: E402


def write_model(root, model_dir, faces, K):
    verts, fcs = scenes.object_mesh(faces)
    m = MeshGaussianModel.from_params(scenes.init_mesh_gaussians(verts, fcs, K=K, seed=5), "cuda", packed_features=True)
    os.makedirs(os.path.join(model_dir, "point_cloud", "iteration_1"), exist_ok=True)
    io_ply.save_mesh_model(os.path.join(model_dir, "point_cloud", "iteration_1", "point_cloud.ply"), m)
    cfg = argparse.Namespace(sh_degree=3, source_path=root, model_path=model_dir, images="images", resolution=-1,
                             white_background=False, data_device="cuda", eval=True, num_splats=[K], meshes=[], gs_type="gs_mesh")
    with open(os.path.join(model_dir, "cfg_args"), "w") as f:
        f.write(str(cfg))
    return m._scale.shape[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--views", type=int, default=200)
    ap.add_argument("--faces", type=int, default=200_000)
    ap.add_argument("--num_splats", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scripts_cli_eval.py needs a CUDA device")
    print(train_cli_eval.card(), flush=True)
    root, model_dir = os.path.join(a.out, "scene"), os.path.join(a.out, "model")
    if not os.path.exists(os.path.join(root, "transforms_test.json")):
        train_cli_eval.write_scene(root, a.views, a.faces)
    P = write_model(root, model_dir, a.faces, a.num_splats)
    print(f"scene: {a.views} views at 1920x1080; checkpoint: {P} mesh-Gaussians", flush=True)
    if not a.bench:
        return
    times = {}
    orig_frames, orig_gt = cli_render.render_frames, cli_render.write_ground_truth

    def timed_frames(*args, **kw):
        torch.cuda.synchronize()
        t = time.perf_counter()
        n = orig_frames(*args, **kw)
        torch.cuda.synchronize()
        times["program"].append((time.perf_counter() - t, n))
        return n

    cli_render.render_frames, cli_render.write_ground_truth = timed_frames, lambda *x, **k: None
    argv = ["-m", model_dir, "--skip_test", "--quiet"]
    args = cli_render.combined_args(render_time_animated.build_parser(), argv)
    sc = cli_render.load_views(args, torch.device("cuda"))
    cams = sc.train_cameras
    model, _ = cli_render.load_model("gs_mesh", os.path.join(model_dir, "point_cloud", "iteration_1", "point_cloud.ply"), 3, "cuda")
    bg = torch.zeros(3, device="cuda")
    frames_dir = os.path.join(a.out, "bare")
    os.makedirs(frames_dir, exist_ok=True)
    cli_render.load_views = lambda *x: sc                        # the scene is loaded once, outside the clock

    def bare():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = NativeRenderer(model, cams[0].image_width, cams[0].image_height)
        tt = render_time_animated.sweep_times(len(cams))
        with torch.no_grad(), io_image.ImageSink(cams[0].image_height, cams[0].image_width) as sink:
            for i, c in enumerate(cams):
                sink.write(r.render(c, bg, vertices=scenes.transform_hotdog_fly(model.vertices, tt[i]))[0],
                           os.path.join(frames_dir, f"{i:05d}.png"))
        torch.cuda.synchronize()
        times["bare"].append((time.perf_counter() - t0, len(cams)))

    times["program"], times["bare"] = [], []
    render_time_animated.main(argv)      # warm-up of both arms
    bare()
    times["program"], times["bare"] = [], []
    for _ in range(a.runs):
        render_time_animated.main(argv)
        bare()
    fps = {k: [n / t for t, n in v] for k, v in times.items()}
    med = {k: statistics.median(v) for k, v in fps.items()}
    for k in ("program", "bare"):
        print(f"{k:8s} frames/s per run: {', '.join(f'{x:.2f}' for x in fps[k])}  median {med[k]:.2f}")
    print(f"program overhead against the bare loop: {100.0 * (med['bare'] / med['program'] - 1.0):+.2f} % "
          f"({len(cams)} frames per run, {a.runs} runs per arm)")


if __name__ == "__main__":
    main()
