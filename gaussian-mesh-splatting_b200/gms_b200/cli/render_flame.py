"""python -m gms_b200.cli.render_flame -m <output> [--iteration N] [--animated] [--skip_train] [--skip_test]: the
reference's scripts/render_flame.py on the native FLAME model and renderer.

A gs_flame checkpoint is loaded with its FLAME model (render.load_flame: FlameCheckpoint and NativeFlame.from_checkpoint),
and the mesh is posed once (gms_flame_lbs_forward) then drawn from every view of a split (gms_flame_render_frame):
- without --animated, at the checkpoint's FLAME parameters, into {model}/{split}/ours_{it}/renders_{gs_type}/ with the
  ground truth in .../gt/;
- with --animated, at the checkpoint's parameters with expression coefficients 0, 5, 7 and 9 set to 2, into
  .../flame_animated/, no ground truth, and that pose's mesh is written first to
  .../flame_animated/{it}_flame_render_vertices.pt: an OBJ text file (write_mesh_obj's format) despite its name.
--seed plays safe_state's role, as in the other programs.

Quirk kept from the script: the background is always white, whatever -w says."""
from __future__ import annotations

import os

import torch

from .. import io_obj
from ..render import FlameRenderer
from . import render

ANIMATED_EXPRESSIONS = (0, 5, 7, 9)     # expression coefficients --animated sets to 2


def output_dirs(model_path: str, name: str, iteration: int, gs_type: str, animated: bool):
    """(frame directory, ground-truth directory or None, vertex file or None) of a split."""
    if animated:
        d, _ = render.split_dirs(model_path, name, iteration, "flame_animated", gt=False)
        return d, None, os.path.join(d, f"{iteration}_flame_render_vertices.pt")
    return render.split_dirs(model_path, name, iteration, f"renders_{gs_type}") + (None,)


def build_parser():
    p = render.script_parser()
    p.add_argument("--iteration", default=-1, type=int)
    p.add_argument("--gs_type", type=str, default="gs_flame")
    p.add_argument("--num_splats", nargs="+", type=int, default=5)
    p.add_argument("--skip_train", action="store_true")
    p.add_argument("--skip_test", action="store_true")
    p.add_argument("--animated", action="store_true")
    p.add_argument("--quiet", action="store_true")
    p.add_argument("--seed", type=int, default=0)
    return p


def animated_expression(exp: torch.Tensor) -> torch.Tensor:
    """render_set_animated's expression: a copy of the checkpoint's [1,n_exp] with coefficients 0, 5, 7, 9 set to 2."""
    out = exp.clone()
    for k in ANIMATED_EXPRESSIONS:
        out[0, k] = 2
    return out


def main(argv=None) -> dict:
    parser = build_parser()
    args, dev, iteration, ply = render.prepare(parser, argv, "render_flame")
    model, flame = render.load_flame(ply, args.sh_degree, dev)
    sc = render.load_views(args, dev)
    bg = render.background(True, dev)
    done = {}
    with torch.no_grad():
        if args.animated:
            vertices = model.driver_vertices(flame, expression_params=animated_expression(model._flame_exp))
        else:
            vertices = model.driver_vertices(flame)
        for name, cams, images in render.splits(args, sc):
            frames, gts, mesh = output_dirs(args.model_path, name, iteration, args.gs_type, args.animated)
            if mesh is not None:
                os.makedirs(frames, exist_ok=True)
                io_obj.write_obj(mesh, vertices, model.faces)
            done[name] = render.render_frames(model, FlameRenderer, cams,
                                              lambda r, idx, cam: r.render(cam, bg, vertices=vertices, antialiasing=args.antialiasing)[0],
                                              frames, gts, images, dev, name)
    return {"iteration": iteration, "views": done}


if __name__ == "__main__":
    main()
