"""python -m gms_b200.cli.render_multi_mesh -m <output> [--iteration N] [--skip_train] [--skip_test]: the reference's
scripts/render_multi_mesh.py on the native renderer.

A gs_multi_mesh checkpoint (point_cloud.ply + model_params.pt) is loaded as one segmented model (render.load_multi_mesh,
one mesh segment per mesh whatever their splat counts) and every view of a split is drawn into
{model}/{split}/ours_{it}/renders/{idx:05d}.png, the ground truth into .../gt/.  --gs_type, --num_splats and --meshes are
accepted and change nothing drawn, as in the script.  --seed plays safe_state's role, as in the other programs.

Quirk kept from the script: the renders go to renders/, not renders_{gs_type}/, so metrics.py (and cli.metrics) never
find them; `cli.render --gs_type gs_multi_mesh` writes the same images where they do."""
from __future__ import annotations

import torch

from ..render import NativeRenderer
from . import render


FRAMES = "renders"


def build_parser():
    p = render.script_parser()
    p.add_argument("--iteration", default=-1, type=int)
    p.add_argument("--gs_type", type=str, default="gs")
    p.add_argument("--skip_train", action="store_true")
    p.add_argument("--skip_test", action="store_true")
    p.add_argument("--quiet", action="store_true")
    p.add_argument("--num_splats", nargs="+", type=int, default=[])
    p.add_argument("--meshes", nargs="+", type=str, default=[])
    p.add_argument("--seed", type=int, default=0)
    return p


def main(argv=None) -> dict:
    parser = build_parser()
    args, dev, iteration, ply = render.prepare(parser, argv, "render_multi_mesh")
    model = render.load_multi_mesh(ply, args.sh_degree, dev)
    sc = render.load_views(args, dev)
    bg = render.background(args.white_background, dev)
    done = {}
    with torch.no_grad():
        for name, cams, images in render.splits(args, sc):
            done[name] = render.render_frames(model, NativeRenderer, cams,
                                              lambda r, idx, cam: r.render(cam, bg, antialiasing=args.antialiasing)[0],
                                              *render.split_dirs(args.model_path, name, iteration, FRAMES), images, dev, name)
    return {"iteration": iteration, "views": done}


if __name__ == "__main__":
    main()
