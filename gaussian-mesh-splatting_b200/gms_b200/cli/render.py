"""python -m gms_b200.cli.render -m <output> [--iteration N] [--gs_type gs_mesh|gs_flat|gs|gs_points|gs_multi_mesh|gs_flame]
[--skip_train] [--skip_test] [--antialiasing]: the reference's scripts/render.py on the native renderers.

The model directory's cfg_args is merged with the command line as get_combined_args does (so --gs_type defaults to gs_flat
whatever the run trained, as in the reference).  The scene is loaded unshuffled; every view of a split is rendered with the
white or black background and written to {model}/{split}/ours_{iter}/renders_{gs_type}/{idx:05d}.png through ImageSink,
and its ground truth to .../gt/{idx:05d}.png.  gs_multi_mesh is drawn as one segmented model (load_multi_mesh); gs_flame
at its checkpoint pose, the FLAME model rebuilt from the checkpoint (load_flame), over the background -w picks.  The
ground-truth PNGs are the resident 8-bit images themselves: save_image of byte / 255 gives the byte back for all 256
values, so they are what the reference writes.  render_frames is the frame loop the other render programs share."""
from __future__ import annotations

import os
import sys
from argparse import ArgumentParser
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from .. import dataset, io_image, io_ply
from ..flame import NativeFlame
from ..model import FlameCheckpoint, FreeGaussianModel, MeshGaussianModel, MultiMeshGaussianModel, PointsModel
from ..render import FlameRenderer, NativeFreeRenderer, NativeRenderer, PointsRenderer
from . import options

GS_TYPES = ("gs_mesh", "gs_flat", "gs", "gs_points", "gs_multi_mesh", "gs_flame")


def script_parser() -> ArgumentParser:
    """What every render script declares first: ModelParams(parser, sentinel=True), then PipelineParams(parser)."""
    p = ArgumentParser(description="Testing script parameters")
    options.add_group(p, "Loading Parameters", options.MODEL_PARAMS, fill_none=True)
    options.add_group(p, "Pipeline Parameters", options.PIPELINE_PARAMS)
    return p


def build_parser() -> ArgumentParser:
    p = script_parser()
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
    if gs_type == "gs_multi_mesh":
        return load_multi_mesh(ply, sh_degree, device), NativeRenderer
    if gs_type == "gs_flame":
        model, flame = load_flame(ply, sh_degree, device)
        model.vertices = model.driver_vertices(flame)
        return model, FlameRenderer
    return FreeGaussianModel.from_checkpoint(ply, gs_type, device, active_sh_degree=sh_degree), NativeFreeRenderer


def load_multi_mesh(ply: str, sh_degree: int, device) -> MultiMeshGaussianModel:
    """A gs_multi_mesh checkpoint (point_cloud.ply + model_params.pt) as one segmented model: one mesh segment per mesh,
    whatever their splat counts."""
    return MultiMeshGaussianModel.from_mesh_params(io_ply.load_multi_mesh_model(ply), device, sh_degree=sh_degree,
                                                   active_sh_degree=sh_degree, packed_features=True, segmented=True)


def load_flame(ply: str, sh_degree: int, device):
    """(FlameCheckpoint, NativeFlame) of a gs_flame checkpoint (point_cloud.ply + flame_params.pt): the FLAME model is
    rebuilt from the checkpoint's own `point_cloud` entry, so no FLAME model file is needed."""
    ckpt = io_ply.load_flame_model(ply)
    return FlameCheckpoint(ckpt, device, active_sh_degree=sh_degree), NativeFlame.from_checkpoint(ckpt["point_cloud"], device)


def _write_png_u8(img_u8: np.ndarray, path: str) -> None:
    H, W, Cn = img_u8.shape
    rows = np.concatenate([np.zeros((H, 1), np.uint8), img_u8.reshape(H, W * Cn)], axis=1)
    with open(path, "wb") as f:
        f.write(io_image.encode_png(rows.tobytes(), W, H, Cn))


def write_ground_truth(images, gts_path: str) -> None:
    """The resident uint8 [H,W,3] images as gts_path/{idx:05d}.png, encoded on host threads (each read-back waits for
    the work queued before it)."""
    with ThreadPoolExecutor(max(2, min(16, (os.cpu_count() or 4) // 4))) as ex:
        jobs = [ex.submit(_write_png_u8, img.cpu().numpy(), os.path.join(gts_path, f"{idx:05d}.png"))
                for idx, img in enumerate(images)]
        for j in jobs:
            j.result()


def render_frames(model, renderer_cls, cams, draw, render_path: str, gts_path: str = None, images=None, device=None,
                  what: str = "frames") -> int:
    """The frame loop every render program shares.  Frame idx is draw(renderer, idx, cams[idx]) -> image [3,H,W], written
    to render_path/{idx:05d}.png; there is one renderer and one ImageSink per image size, and no host synchronisation after
    the first frame.  With gts_path, the ground truth `images` leave the device once every frame is queued.  A sync-free
    render whose binning capacity was predicted too small draws only the background: if any did, every frame is drawn
    again, each view now sized from its true N (a view is keyed by its camera's uid)."""
    os.makedirs(render_path, exist_ok=True)
    if gts_path is not None:
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
                sinks[size].write(draw(renderers[size], idx, cam), os.path.join(render_path, f"{idx:05d}.png"))
            if attempt == 0 and gts_path is not None:
                write_ground_truth(images, gts_path)
        finally:
            for s in sinks.values():
                s.close()           # (waits for every frame: the renders before them are done)
        for r in renderers.values():
            r._harvest()
        if sum(r.overflows for r in renderers.values()) == start:
            break
        if attempt == 1:
            raise RuntimeError(f"renders of {what} overflowed their binning capacity twice")
    return len(cams)


def split_dirs(model_path: str, name: str, iteration: int, frames: str, gt: bool = True):
    """(frame directory, ground-truth directory or None) of a split: {model}/{split}/ours_{iteration}/{frames} and .../gt."""
    out = os.path.join(model_path, name, f"ours_{iteration}")
    return os.path.join(out, frames), (os.path.join(out, "gt") if gt else None)


def render_set(model, renderer_cls, model_path: str, name: str, iteration: int, cams, images, bg, gs_type: str,
               antialiasing: bool, device) -> int:
    """render_set: every view of the split at the model's own pose into renders_{gs_type}/, its ground truth into gt/."""
    return render_frames(model, renderer_cls, cams, lambda r, idx, cam: r.render(cam, bg, antialiasing=antialiasing)[0],
                         *split_dirs(model_path, name, iteration, f"renders_{gs_type}"), images, device, name)


def combined_args(parser: ArgumentParser, argv):
    """get_combined_args on argv (the process's arguments when None)."""
    return options.combined_args(parser, sys.argv[1:] if argv is None else argv)


def device(parser: ArgumentParser, args, prog: str) -> torch.device:
    """The CUDA device the program renders on; refuses --data_device other than cuda."""
    if getattr(args, "data_device", "cuda") != "cuda":
        parser.error(f"--data_device {args.data_device} is not supported: images stay resident on the GPU")
    if not torch.cuda.is_available():
        raise RuntimeError(f"gms_b200.cli.{prog} needs a CUDA device")
    return torch.device("cuda")


def prepare(parser: ArgumentParser, argv, prog: str):
    """A render script's start: get_combined_args, the device, the "Rendering" line and the checkpoint to load ->
    (args, device, iteration, point_cloud.ply path)."""
    args = combined_args(parser, argv)
    dev = device(parser, args, prog)
    if not args.quiet:
        print("Rendering " + args.model_path)
    iteration, ply = checkpoint(args.model_path, args.iteration)
    return args, dev, iteration, ply


def checkpoint(model_path: str, iteration: int):
    """(iteration, point_cloud.ply path): --iteration -1 is the largest saved one (Scene's load_iteration)."""
    if iteration == -1:
        iteration = search_max_iteration(os.path.join(model_path, "point_cloud"))
    return iteration, os.path.join(model_path, "point_cloud", f"iteration_{iteration}", "point_cloud.ply")


def load_views(args, dev):
    """The scene's cameras and resident uint8 images, unshuffled.  Only cameras and images: the gs_mesh reader would also
    rebuild the initial mesh model, which a render does not use.  Nothing is written into the source directory."""
    resolution = -1 if args.resolution is None else args.resolution
    return dataset.load_scene(args.source_path, "gs_flat", bool(args.white_background), bool(args.eval), resolution,
                              args.images or "images", 2, args.seed, shuffle=False, device=dev)


def background(white: bool, dev) -> torch.Tensor:
    return torch.tensor([1.0, 1.0, 1.0] if white else [0.0, 0.0, 0.0], dtype=torch.float32, device=dev)


def splits(args, sc):
    """(name, cameras, images) of the splits the run renders: train unless args.skip_train, then test unless
    args.skip_test."""
    out = []
    if not args.skip_train:
        out.append(("train", sc.train_cameras, sc.train_images))
    if not args.skip_test:
        out.append(("test", sc.test_cameras, sc.test_images))
    return out


def main(argv=None) -> dict:
    parser = build_parser()
    args = combined_args(parser, argv)
    if args.gs_type not in GS_TYPES:
        parser.error(f"--gs_type {args.gs_type} is not supported (supported: {', '.join(GS_TYPES)})")
    dev = device(parser, args, "render")
    if not args.quiet:
        print("Rendering " + args.model_path)
    iteration, ply = checkpoint(args.model_path, args.iteration)
    model, renderer_cls = load_model(args.gs_type, ply, args.sh_degree, dev)
    sc = load_views(args, dev)
    bg = background(args.white_background, dev)
    done = {}
    with torch.no_grad():
        for name, cams, images in splits(args, sc):
            done[name] = render_set(model, renderer_cls, args.model_path, name, iteration, cams, images, bg, args.gs_type,
                                    args.antialiasing, dev)
    return {"iteration": iteration, "views": done}


if __name__ == "__main__":
    main()
