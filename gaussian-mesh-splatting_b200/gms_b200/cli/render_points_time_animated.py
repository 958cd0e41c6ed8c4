"""python -m gms_b200.cli.render_points_time_animated -m <output> [--iteration N] [--skip_train] [--skip_test]: the
reference's scripts/render_points_time_animated.py on the native pseudo-mesh renderer.

A gs_flat checkpoint is loaded as its pseudo-mesh (PointsModel.from_flat_checkpoint) and every view of a split is drawn
with the triangles moved by scenes.transform_hotdog(triangles, t[43]), into
{model}/{split}/ours_{it}/time_animated_gs_points/{idx:05d}.png; the ground truth goes to .../gt/.  --seed plays
safe_state's role, as in the other programs.

Quirk kept from the script: t = torch.linspace(0, 10 pi, n views) (CPU, float32), but EVERY frame is drawn at t[43], so
the frames show one pose from different views.  A split of 1 to 43 views has no t[43]: the script raises IndexError on
it; here the program exits with an error that says so, before anything is rendered."""
from __future__ import annotations

import torch

from .. import scenes
from ..model import PointsModel
from ..render import PointsRenderer
from . import render
from .render_time_animated import sweep_times

FRAME_T = 43        # the index of t every frame uses
FRAMES = "time_animated_gs_points"


def build_parser():
    p = render.script_parser()
    p.add_argument("--iteration", default=-1, type=int)
    p.add_argument("--skip_train", action="store_true")
    p.add_argument("--skip_test", action="store_true")
    p.add_argument("--quiet", action="store_true")
    p.add_argument("--gs_type", type=str, default="gs_points")
    p.add_argument("--num_splats", type=int, default=2)
    p.add_argument("--seed", type=int, default=0)
    return p


def frame_time(n: int) -> torch.Tensor:
    """t[43] of sweep_times(n): the time every frame of an n-view split is drawn at; ValueError when n <= 43."""
    if n <= FRAME_T:
        raise ValueError(f"render_points_time_animated draws every frame at t[{FRAME_T}] of linspace(0, 10 pi, views), so a "
                         f"split needs at least {FRAME_T + 1} views; this one has {n} (the reference script raises IndexError)")
    return sweep_times(n)[FRAME_T]


def main(argv=None) -> dict:
    parser = build_parser()
    args, dev, iteration, ply = render.prepare(parser, argv, "render_points_time_animated")
    sc = render.load_views(args, dev)
    todo = render.splits(args, sc)
    for name, cams, _ in todo:
        if cams:
            try:
                frame_time(len(cams))
            except ValueError as e:
                parser.error(f"{name} split: {e}")
    model = PointsModel.from_flat_checkpoint(ply, dev, active_sh_degree=args.sh_degree)
    bg = render.background(args.white_background, dev)
    done = {}
    with torch.no_grad():
        for name, cams, images in todo:
            tri = scenes.transform_hotdog(model.triangles, frame_time(len(cams))) if cams else None

            def draw(r, idx, cam, tri=tri):
                return r.render(cam, bg, triangles=tri, antialiasing=args.antialiasing)[0]

            done[name] = render.render_frames(model, PointsRenderer, cams, draw,
                                              *render.split_dirs(args.model_path, name, iteration, FRAMES), images, dev, name)
    return {"iteration": iteration, "views": done}


if __name__ == "__main__":
    main()
