"""python -m gms_b200.cli.render_from_mesh_to_mesh -m <output> --target_mesh <mesh.obj> [--iteration N] [--skip_train]
[--skip_test]: the reference's scripts/render_from_mesh_to_mesh.py on the native renderer.

A gs_mesh checkpoint's triangles (vertices[faces]) are morphed into those of a target mesh (read_obj, then
transform_vertices_function with c = 1: (x, -z, y)), face by face.  With n views in a split, frame idx draws
source + morph_step(source, target, n) * idx = source + (target - source) / n * idx from view 0's camera into
{model}/{split}/ours_{it}/from_mesh_to_mesh_animated/{idx:05d}.png, and view idx's ground truth into .../gt/.  The
Gaussians are drawn on the morphed triangles as a triangle soup (vertex 3f + c is corner c of face f), so each frame is
one gms_render_frame with that frame's vertices.  --seed plays safe_state's role, as in the other programs.

Quirk kept from the script: the last frame is idx = n - 1, so the morph stops one step short of the target mesh.
Deliberate differences: --target_mesh replaces the script's hard-coded ../data/ficus/ficus_animate.obj, and a target
whose face count is not the model's is refused before anything is rendered; the OBJ is read by io_obj.read_obj, not
trimesh.load, so vertices are never merged."""
from __future__ import annotations

import dataclasses

import torch

from .. import io_obj
from ..render import NativeRenderer
from . import render


FRAMES = "from_mesh_to_mesh_animated"


def build_parser():
    p = render.script_parser()
    p.add_argument("--iteration", default=-1, type=int)
    p.add_argument("--gs_type", type=str, default="gs_mesh")
    p.add_argument("--num_splats", nargs="+", type=int, default=[2])
    p.add_argument("--skip_train", action="store_true")
    p.add_argument("--skip_test", action="store_true")
    p.add_argument("--quiet", action="store_true")
    p.add_argument("--target_mesh", type=str, required=True, help="OBJ file of the mesh the model's mesh morphs into")
    p.add_argument("--seed", type=int, default=0)
    return p


def transform_vertices_function(vertices: torch.Tensor, c=1) -> torch.Tensor:
    """The script's transform_vertices_function: (x, y, z) -> (x, -z, y) * c, out of place."""
    v = vertices[:, [0, 2, 1]]
    v[:, 1] = -v[:, 1]
    v *= c
    return v


def target_triangles(path: str, device) -> torch.Tensor:
    """float32 [F,3,3]: the target OBJ's triangles after transform_vertices_function, on `device`."""
    v, f = io_obj.read_obj(path)
    return transform_vertices_function(v)[f].to(device)


def morph_step(source: torch.Tensor, target: torch.Tensor, n: int) -> torch.Tensor:
    """The script's diff: (target - source) / n, for a morph over n frames."""
    return (target - source) / n


def morph_triangles(source: torch.Tensor, step: torch.Tensor, idx: int) -> torch.Tensor:
    """The triangles of frame idx: source + step * idx."""
    return source + step * idx


def main(argv=None) -> dict:
    parser = build_parser()
    args, dev, iteration, ply = render.prepare(parser, argv, "render_from_mesh_to_mesh")
    model, _ = render.load_model("gs_mesh", ply, args.sh_degree, dev)
    source = model.vertices.detach()[model.faces].contiguous()
    target = target_triangles(args.target_mesh, dev)
    F = source.shape[0]
    if target.shape[0] != F:
        parser.error(f"--target_mesh {args.target_mesh} has {target.shape[0]} faces; the model's mesh has {F}")
    model.vertices = source.reshape(3 * F, 3)       # the same triangles as a soup
    model.faces = torch.arange(3 * F, dtype=torch.int64, device=dev).reshape(F, 3)
    sc = render.load_views(args, dev)
    bg = render.background(args.white_background, dev)
    done = {}
    with torch.no_grad():
        for name, cams, images in render.splits(args, sc):
            n = len(cams)
            step = morph_step(source, target, n)
            # every frame is drawn from view 0's camera; a uid per frame keeps each frame's binning capacity its own
            frames = [dataclasses.replace(cams[0], uid=(name, "mesh_to_mesh", idx)) for idx in range(n)]

            def draw(r, idx, cam, step=step):
                tri = morph_triangles(source, step, idx)
                return r.render(cam, bg, antialiasing=args.antialiasing, vertices=tri.reshape(3 * F, 3))[0]

            done[name] = render.render_frames(model, NativeRenderer, frames, draw,
                                              *render.split_dirs(args.model_path, name, iteration, FRAMES), images, dev, name)
    return {"iteration": iteration, "views": done}


if __name__ == "__main__":
    main()
