"""python -m gms_b200.cli.render_from_object -m <output> --object_path <mesh.obj> [--scale S] [--skip_train] [--skip_test]:
the reference's scripts/render_from_object.py on the native pseudo-mesh renderer.

The Gaussians of a gs_flat checkpoint (PointsModel.from_flat_checkpoint: their colours and opacities) are drawn on the
triangles of another mesh (object_triangles: the OBJ's triangles / scale, then x -= 0.2), one Gaussian per triangle, into
{model}/{split}/ours_{it}/<basename>/{idx:05d}.png, <basename> being the OBJ's file name up to its first '.'.  No ground
truth is written.  The OBJ must have as many triangles as the checkpoint has Gaussians (the script's renderer needs that
too).  --seed plays safe_state's role, as in the other programs.

Quirk kept from the script: --skip_train is a store_false flag, so the train views are skipped UNLESS it is given (and
giving it renders them).  Deliberate difference: the OBJ is read by io_obj.read_obj, not trimesh.load, so vertices are
never merged; for a triangle soup the triangles are the ones trimesh gives."""
from __future__ import annotations

import os

import torch

from .. import io_obj
from ..model import PointsModel
from ..render import PointsRenderer
from . import render


def build_parser():
    p = render.script_parser()
    p.add_argument("--iteration", default=-1, type=int)
    p.add_argument("--skip_train", action="store_false")
    p.add_argument("--skip_test", action="store_true")
    p.add_argument("--quiet", action="store_true")
    p.add_argument("--gs_type", type=str, default="gs_points")
    p.add_argument("--scale", default=2, type=float)
    p.add_argument("--object_path", default="", type=str)
    p.add_argument("--seed", type=int, default=0)
    return p


def output_name(object_path: str) -> str:
    """The render directory's name: the OBJ's base name up to its first '.'."""
    return os.path.basename(object_path).split(".")[0]


def object_triangles(object_path: str, scale: float, device) -> torch.Tensor:
    """float32 [F,3,3]: the OBJ's triangles on `device`, divided by `scale` there, then x -= 0.2 (the script's order; its
    float64 triangles rounded to float32 are read_obj's float32 vertices)."""
    v, f = io_obj.read_obj(object_path)
    tri = v[f].to(device) / scale
    tri[:, :, 0] -= 0.2
    return tri


def main(argv=None) -> dict:
    parser = build_parser()
    args, dev, iteration, ply = render.prepare(parser, argv, "render_from_object")
    model = PointsModel.from_flat_checkpoint(ply, dev, active_sh_degree=args.sh_degree)
    tri = object_triangles(args.object_path, args.scale, dev)
    if tri.shape[0] != model.triangles.shape[0]:
        parser.error(f"{args.object_path} has {tri.shape[0]} triangles; the checkpoint has {model.triangles.shape[0]} Gaussians "
                     "(one per triangle)")
    sc = render.load_views(args, dev)
    bg = render.background(args.white_background, dev)
    done = {}
    with torch.no_grad():
        for name, cams, _ in render.splits(args, sc):
            out, _ = render.split_dirs(args.model_path, name, iteration, output_name(args.object_path), gt=False)
            done[name] = render.render_frames(
                model, PointsRenderer, cams, lambda r, idx, cam: r.render(cam, bg, triangles=tri, antialiasing=args.antialiasing)[0],
                out, device=dev, what=name)
    return {"iteration": iteration, "views": done}


if __name__ == "__main__":
    main()
