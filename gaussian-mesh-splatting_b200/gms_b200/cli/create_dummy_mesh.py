"""python -m gms_b200.cli.create_dummy_mesh --pseudomesh_path <triangles.pt> [--scale S] [--alpha A]: the reference's
scripts/create_dummy_mesh.py.

The pseudo-mesh's [P,3,3] triangles (save_pseudomesh's triangles.pt) become 3P points, times --scale, in float32 as the script
computes them.  Their alpha shape (alpha_shape.alpha_shape) and per-point normals (alpha_shape.estimate_normals with the
script's radius 0.1 and max_nn 30) are written to {dirname(--pseudomesh_path)}/mesh_alpha_0_003.obj.  The file name is the
script's and is the same for every --alpha, a quirk kept on purpose.  An empty alpha shape writes an empty OBJ and says that
no tetrahedron met alpha.  cli.edit_pseudomesh takes the file as --mesh_path.

Deliberate differences, all on the GPU and in float64:
- vertex and face order: vertices in ascending point index, faces with ascending vertex indices in lexicographic order
  (open3d's follow Qhull's facet order);
- the normal sign: n.(x - mean of the points) >= 0 (outward on star-shaped objects), where open3d's is arbitrary;
- OBJ text: io_obj.write_obj's `v` / `vn` / `f a//a b//b c//c` records with %f, not trimesh's export (no header comment);
- vertices are not merged beyond exact duplicates."""
from __future__ import annotations

import os
import sys
from argparse import ArgumentParser

import torch

from .. import io_obj
from ..alpha_shape import alpha_shape, estimate_normals

NORMAL_RADIUS, NORMAL_MAX_NN = 0.1, 30      # KDTreeSearchParamHybrid(radius=0.1, max_nn=30)
OUTPUT_NAME = "mesh_alpha_0_003.obj"


def build_parser():
    p = ArgumentParser(description="Testing script parameters")
    p.add_argument("--pseudomesh_path", type=str)
    p.add_argument("--scale", default=2, type=int)
    p.add_argument("--alpha", default=0.003, type=float)
    return p


def output_path(pseudomesh_path: str) -> str:
    return os.path.join(os.path.dirname(pseudomesh_path), OUTPUT_NAME)


def main(argv=None) -> dict:
    parser = build_parser()
    args = parser.parse_args(sys.argv[1:] if argv is None else argv)
    if args.pseudomesh_path is None:
        parser.error("--pseudomesh_path is needed")
    if not torch.cuda.is_available():
        raise RuntimeError("gms_b200.cli.create_dummy_mesh needs a CUDA device")
    p = torch.load(args.pseudomesh_path, map_location="cuda", weights_only=True)
    if p.dim() != 3 or p.shape[1:] != (3, 3):
        parser.error(f"--pseudomesh_path {args.pseudomesh_path} must hold [P,3,3] triangles; got {tuple(p.shape)}")
    xyz = (p.reshape(p.shape[0] * 3, 3) * args.scale).float().contiguous()
    normals = estimate_normals(xyz, NORMAL_RADIUS, NORMAL_MAX_NN)
    vertices, faces, index = alpha_shape(xyz, args.alpha)
    out = output_path(args.pseudomesh_path)
    io_obj.write_obj(out, vertices, faces, normals[index])
    if faces.shape[0] == 0:
        print(f"No tetrahedron has a circumradius <= alpha = {args.alpha}: wrote an empty mesh to {out}")
    else:
        print(f"Alpha shape: {vertices.shape[0]} vertices, {faces.shape[0]} faces -> {out}")
    return {"path": out, "points": xyz.shape[0], "vertices": int(vertices.shape[0]), "faces": int(faces.shape[0])}


if __name__ == "__main__":
    main()
