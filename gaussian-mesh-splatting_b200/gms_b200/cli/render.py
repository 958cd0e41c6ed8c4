"""python -m gms_b200.cli.render -m <output> [--iteration N] [--gs_type gs_mesh|gs_flat|gs|gs_points] [--skip_train]
[--skip_test] [--antialiasing]: the reference's scripts/render.py on the native renderers.

The model directory's cfg_args is merged with the command line as get_combined_args does (so --gs_type defaults to gs_flat
whatever the run trained, as in the reference).  The scene is loaded unshuffled; every view of a split is rendered with the
white or black background and written to {model}/{split}/ours_{iter}/renders_{gs_type}/{idx:05d}.png through ImageSink,
and its ground truth to .../gt/{idx:05d}.png.  The ground-truth PNGs are the resident 8-bit images themselves: save_image
of byte / 255 gives the byte back for all 256 values, so they are what the reference writes."""
from __future__ import annotations

import os
import sys
from argparse import ArgumentParser
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from .. import dataset, io_image, io_ply
from ..model import FreeGaussianModel, MeshGaussianModel, PointsModel
from ..render import NativeFreeRenderer, NativeRenderer, PointsRenderer
from . import options

GS_TYPES = ("gs_mesh", "gs_flat", "gs", "gs_points")


def build_parser() -> ArgumentParser:
    p = ArgumentParser(description="Testing script parameters")
    options.add_group(p, "Loading Parameters", options.MODEL_PARAMS, fill_none=True)
    options.add_group(p, "Pipeline Parameters", options.PIPELINE_PARAMS)
    p.add_argument("--iteration", default=-1, type=int)
    p.add_argument("--gs_type", type=str, default="gs_flat")
    p.add_argument("--num_splats", nargs="+", type=int, default=[2])
    p.add_argument("--skip_train", action="store_true")
    p.add_argument("--skip_test", action="store_true")
    p.add_argument("--quiet", action="store_true")
    p.add_argument("--seed", type=int, default=0)
    return p


def search_max_iteration(folder: str) -> int:
    """searchForMaxIteration (utils/system_utils.py): the largest N of the iteration_N entries."""
    return max(int(f.split("_")[-1]) for f in os.listdir(folder))


def load_model(gs_type: str, ply: str, sh_degree: int, device):
    """The checkpoint and the renderer class that draws it (load_ply sets the active SH degree to the maximum)."""
    if gs_type == "gs_mesh":
        m = MeshGaussianModel.from_params(io_ply.load_mesh_model(ply), device, sh_degree=sh_degree, active_sh_degree=sh_degree,
                                          packed_features=True)
        return m, NativeRenderer
    if gs_type == "gs_points":
        return PointsModel.from_flat_checkpoint(ply, device, active_sh_degree=sh_degree), PointsRenderer
    return FreeGaussianModel.from_checkpoint(ply, gs_type, device, active_sh_degree=sh_degree), NativeFreeRenderer


def _write_png_u8(img_u8: np.ndarray, path: str) -> None:
    H, W, Cn = img_u8.shape
    rows = np.concatenate([np.zeros((H, 1), np.uint8), img_u8.reshape(H, W * Cn)], axis=1)
    with open(path, "wb") as f:
        f.write(io_image.encode_png(rows.tobytes(), W, H, Cn))


def render_set(model, renderer_cls, model_path: str, name: str, iteration: int, cams, images, bg, gs_type: str,
               antialiasing: bool, device) -> int:
    """render_set: one renderer and one ImageSink per image size; the ground truth leaves the device once every render of
    the split is queued.  A sync-free render whose binning capacity was predicted too small draws only the background: if
    any did, the split is rendered again, every view now sized from its true N."""
    render_path = os.path.join(model_path, name, f"ours_{iteration}", f"renders_{gs_type}")
    gts_path = os.path.join(model_path, name, f"ours_{iteration}", "gt")
    os.makedirs(render_path, exist_ok=True)
    os.makedirs(gts_path, exist_ok=True)
    renderers = {}
    for attempt in range(2):
        start = sum(r.overflows for r in renderers.values())
        sinks = {}
        try:
            for idx, cam in enumerate(cams):
                size = (int(cam.image_width), int(cam.image_height))
                if size not in renderers:
                    renderers[size] = renderer_cls(model, *size)
                if size not in sinks:
                    sinks[size] = io_image.ImageSink(size[1], size[0], device=device)
                image = renderers[size].render(cam, bg, antialiasing=antialiasing)[0]
                sinks[size].write(image, os.path.join(render_path, f"{idx:05d}.png"))
            if attempt == 0:
                with ThreadPoolExecutor(max(2, min(16, (os.cpu_count() or 4) // 4))) as ex:
                    jobs = [ex.submit(_write_png_u8, img.cpu().numpy(), os.path.join(gts_path, f"{idx:05d}.png"))
                            for idx, img in enumerate(images)]
                    for j in jobs:
                        j.result()
        finally:
            for s in sinks.values():
                s.close()           # (waits for every frame: the renders before them are done)
        for r in renderers.values():
            r._harvest()
        if sum(r.overflows for r in renderers.values()) == start:
            break
        if attempt == 1:
            raise RuntimeError(f"renders of {name} overflowed their binning capacity twice")
    return len(cams)


def main(argv=None) -> dict:
    parser = build_parser()
    args = options.combined_args(parser, sys.argv[1:] if argv is None else argv)
    if args.gs_type not in GS_TYPES:
        parser.error(f"--gs_type {args.gs_type} is not supported (supported: {', '.join(GS_TYPES)})")
    if getattr(args, "data_device", "cuda") != "cuda":
        parser.error(f"--data_device {args.data_device} is not supported: images stay resident on the GPU")
    if not torch.cuda.is_available():
        raise RuntimeError("gms_b200.cli.render needs a CUDA device")
    dev = torch.device("cuda")
    if not args.quiet:
        print("Rendering " + args.model_path)
    iteration = args.iteration
    if iteration == -1:
        iteration = search_max_iteration(os.path.join(args.model_path, "point_cloud"))
    ply = os.path.join(args.model_path, "point_cloud", f"iteration_{iteration}", "point_cloud.ply")
    model, renderer_cls = load_model(args.gs_type, ply, args.sh_degree, dev)
    resolution = -1 if args.resolution is None else args.resolution
    # cameras and images only: the gs_mesh reader would also rebuild the initial mesh model, which a render does not use
    sc = dataset.load_scene(args.source_path, "gs_flat", bool(args.white_background), bool(args.eval), resolution,
                            args.images or "images", args.num_splats[0], args.seed, shuffle=False, device=dev)
    bg = torch.tensor([1.0, 1.0, 1.0] if args.white_background else [0.0, 0.0, 0.0], dtype=torch.float32, device=dev)
    done = {}
    with torch.no_grad():
        if not args.skip_train:
            done["train"] = render_set(model, renderer_cls, args.model_path, "train", iteration, sc.train_cameras, sc.train_images,
                                       bg, args.gs_type, args.antialiasing, dev)
        if not args.skip_test:
            done["test"] = render_set(model, renderer_cls, args.model_path, "test", iteration, sc.test_cameras, sc.test_images,
                                      bg, args.gs_type, args.antialiasing, dev)
    return {"iteration": iteration, "views": done}


if __name__ == "__main__":
    main()
