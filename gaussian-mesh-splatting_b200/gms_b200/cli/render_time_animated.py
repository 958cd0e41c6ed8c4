"""python -m gms_b200.cli.render_time_animated -m <output> [--iteration N] [--skip_train] [--skip_test]: the reference's
scripts/render_time_animated.py on the native renderer.

A gs_mesh checkpoint is loaded (whatever --gs_type says, as in the script; --gs_type and --num_splats are accepted and
change nothing drawn) and every view idx of a split is drawn with the mesh moved by scenes.transform_hotdog_fly(vertices,
t[idx]), t = sweep_times(n views), into {model}/{split}/ours_{it}/time_animated/{idx:05d}.png; the ground truth goes to
.../gt/.  Each frame is one gms_render_frame at that frame's vertices (NativeRenderer.render(vertices=...)), with no host
synchronisation after the first.  --seed plays safe_state's role, as in the other programs.  The four other transforms
the script defines are never called by it and are not provided."""
from __future__ import annotations

import torch

from .. import scenes
from ..render import NativeRenderer
from . import render


FRAMES = "time_animated"


def build_parser():
    p = render.script_parser()
    p.add_argument("--iteration", default=-1, type=int)
    p.add_argument("--gs_type", type=str, default="gs_mesh")
    p.add_argument("--num_splats", nargs="+", type=int, default=[2])
    p.add_argument("--skip_train", action="store_true")
    p.add_argument("--skip_test", action="store_true")
    p.add_argument("--quiet", action="store_true")
    p.add_argument("--seed", type=int, default=0)
    return p


def sweep_times(n: int) -> torch.Tensor:
    """The script's t: torch.linspace(0, 10 pi, n) on the CPU in float32; frame idx is drawn at t[idx]."""
    return torch.linspace(0, 10 * torch.pi, n)


def main(argv=None) -> dict:
    parser = build_parser()
    args, dev, iteration, ply = render.prepare(parser, argv, "render_time_animated")
    model, _ = render.load_model("gs_mesh", ply, args.sh_degree, dev)
    sc = render.load_views(args, dev)
    bg = render.background(args.white_background, dev)
    done = {}
    with torch.no_grad():
        for name, cams, images in render.splits(args, sc):
            t = sweep_times(len(cams))

            def draw(r, idx, cam, t=t):
                return r.render(cam, bg, antialiasing=args.antialiasing, vertices=scenes.transform_hotdog_fly(model.vertices, t[idx]))[0]

            done[name] = render.render_frames(model, NativeRenderer, cams, draw,
                                              *render.split_dirs(args.model_path, name, iteration, FRAMES), images, dev, name)
    return {"iteration": iteration, "views": done}


if __name__ == "__main__":
    main()
