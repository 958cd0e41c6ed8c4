"""python -m gms_b200.cli.save_pseudomesh --model_path <output> [--iteration N] [--scale S] [--save_faces]
[--save_vertices]: the reference's scripts/save_pseudomesh.py.

A gs_flat checkpoint's pseudo-mesh (PointsModel.from_flat_checkpoint: one triangle per Gaussian, built on the GPU) is
written to {model}/pseudomesh_info/ours_{it}/: triangles.pt (the [P,3,3] triangles, on the device, as the script saves
them), faces.pt with --save_faces (float32 [P,3] = 0 .. 3P-1, torch.range's values and dtype), vertices.pt with
--save_vertices (the [3P,3] triangle soup) and scale_{scale}.obj (io_obj.write_obj of the soup times --scale:
write_simple_obj's text).  The script reads no cfg_args and has no --seed; neither does this program."""
from __future__ import annotations

import os
import sys
from argparse import ArgumentParser

import torch

from .. import io_obj
from ..model import PointsModel
from . import render


def build_parser():
    p = ArgumentParser(description="Testing script parameters")
    p.add_argument("--model_path", type=str)
    p.add_argument("--iteration", default=-1, type=int)
    p.add_argument("--sh_degree", default=3, type=int)
    p.add_argument("--scale", default=2, type=int)
    p.add_argument("--save_faces", action="store_true")
    p.add_argument("--save_vertices", action="store_true")
    return p


def output_dir(model_path: str, iteration: int) -> str:
    return os.path.join(model_path, "pseudomesh_info", f"ours_{iteration}")


def soup_faces(P: int) -> torch.Tensor:
    """torch.range(0, 3P - 1).reshape(P, 3): float32 face indices of the triangle soup."""
    return torch.arange(3 * P, dtype=torch.float32).reshape(P, 3)


def main(argv=None) -> dict:
    parser = build_parser()
    args = parser.parse_args(sys.argv[1:] if argv is None else argv)
    if args.model_path is None:
        parser.error("--model_path is needed")
    if not torch.cuda.is_available():
        raise RuntimeError("gms_b200.cli.save_pseudomesh needs a CUDA device")
    print("Pseudomesh info " + args.model_path)
    iteration, ply = render.checkpoint(args.model_path, args.iteration)
    print("Loading trained model at iteration {}".format(iteration))
    out = output_dir(args.model_path, iteration)
    os.makedirs(out, exist_ok=True)
    triangles = PointsModel.from_flat_checkpoint(ply, "cuda", active_sh_degree=args.sh_degree).triangles
    P = triangles.shape[0]
    torch.save(triangles, os.path.join(out, "triangles.pt"))
    faces = soup_faces(P)
    vertices = triangles.reshape(P * 3, 3)
    if args.save_faces:
        torch.save(faces, os.path.join(out, "faces.pt"))
    if args.save_vertices:
        torch.save(vertices, os.path.join(out, "vertices.pt"))
    io_obj.write_obj(os.path.join(out, f"scale_{args.scale}.obj"), vertices * args.scale, faces)
    return {"iteration": iteration, "path": out, "triangles": P}


if __name__ == "__main__":
    main()
