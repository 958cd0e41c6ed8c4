"""python -m gms_b200.cli.edit_pseudomesh --triangle_soup_path <soup.obj> --mesh_path <mesh.obj> --edited_mesh_path
<edited.obj> --save_dir <dir> [--scale S]: the reference's scripts/edit_pseudomesh_based_on_estimated_mesh.py.

Every triangle of the pseudo-mesh (a triangle soup, e.g. save_pseudomesh's OBJ) is bound to the nearest face of the mesh
(expansion.bind_pseudomesh, on the GPU) and re-posed on the edited mesh (expansion.repose_pseudomesh).  Written to
--save_dir: edited_triangles.pt (the [P,3,3] triangles, on the device, as the script saves them) and
scale_{scale}_edited.obj (io_obj.write_obj of the re-posed soup times --scale: write_simple_obj's text).

Deliberate differences: the OBJ files are read by io_obj.read_obj, not trimesh.load, so vertices are never merged; the
edited mesh must have the mesh's faces (the script pairs their faces by index and assumes it) and is refused otherwise;
--save_dir is created when missing."""
from __future__ import annotations

import os
import sys
from argparse import ArgumentParser

import torch

from .. import expansion, io_obj


def build_parser():
    p = ArgumentParser(description="Testing script parameters")
    p.add_argument("--triangle_soup_path", type=str)
    p.add_argument("--mesh_path", type=str)
    p.add_argument("--edited_mesh_path", type=str)
    p.add_argument("--save_dir", type=str)
    p.add_argument("--scale", default=1, type=int)
    return p


def read_triangles(path: str) -> torch.Tensor:
    """float32 [F,3,3]: an OBJ's triangles (trimesh.load(path).triangles, without vertex merging)."""
    v, f = io_obj.read_obj(path)
    return v[f]


def main(argv=None) -> dict:
    parser = build_parser()
    args = parser.parse_args(sys.argv[1:] if argv is None else argv)
    for k in ("triangle_soup_path", "mesh_path", "edited_mesh_path", "save_dir"):
        if getattr(args, k) is None:
            parser.error(f"--{k} is needed")
    if not torch.cuda.is_available():
        raise RuntimeError("gms_b200.cli.edit_pseudomesh needs a CUDA device")
    v, f = io_obj.read_obj(args.mesh_path)
    ve, fe = io_obj.read_obj(args.edited_mesh_path)
    if not torch.equal(f, fe) or ve.shape != v.shape:
        parser.error(f"--edited_mesh_path {args.edited_mesh_path} must have the faces of --mesh_path {args.mesh_path} "
                     f"({v.shape[0]} vertices, {f.shape[0]} faces); it has {ve.shape[0]} vertices, {fe.shape[0]} faces")
    dev = torch.device("cuda")
    binding = expansion.bind_pseudomesh(read_triangles(args.triangle_soup_path).to(dev), v.to(dev), f.to(dev))
    edited = expansion.repose_pseudomesh(binding, ve.to(dev))
    os.makedirs(args.save_dir, exist_ok=True)
    torch.save(edited, os.path.join(args.save_dir, "edited_triangles.pt"))
    io_obj.write_obj(os.path.join(args.save_dir, f"scale_{args.scale}_edited.obj"), *io_obj.triangle_soup(edited * args.scale))
    return {"triangles": edited.shape[0], "degenerate_faces": binding.n_degenerate}


if __name__ == "__main__":
    main()
