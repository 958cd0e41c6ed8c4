"""The small part of Wavefront OBJ the mesh-driven pseudo-mesh workflow exchanges with an editor (README "Pseudomesh/Triangle
Soup and modifications"): the driving mesh read in, its edited pose read back, and edited pseudo-meshes written out.

    read_obj(path)  -> vertices float32 [V,3], faces int64 [F,3]   (`v` and `f` records only)
    write_obj(path, vertices, faces[, normals])                   (scripts/save_pseudomesh.py:52-59, write_simple_obj;
                                                                   with normals, the dummy mesh of cli.create_dummy_mesh)
"""
from __future__ import annotations

import numpy as np
import torch


def read_obj(path: str):
    """`v x y z [w]` and `f` records of an OBJ file; every other record is ignored.  A face corner may be written `a`, `a/b`,
    `a//c` or `a/b/c` (only the vertex index `a` is used), 1-based or negative (relative to the vertices read so far).
    Polygons are fan-triangulated, (c0, c1, c2), (c0, c2, c3), ..., and faces keep the file's order.
    Returns (vertices float32 [V,3], faces int64 [F,3]) as CPU tensors."""
    verts, faces = [], []
    with open(path, "r") as fh:
        for ln, line in enumerate(fh, 1):
            parts = line.split()
            if not parts:
                continue
            if parts[0] == "v":
                if len(parts) < 4:
                    raise ValueError(f"{path}:{ln}: a vertex needs three coordinates")
                verts.append([float(x) for x in parts[1:4]])
            elif parts[0] == "f":
                if len(parts) < 4:
                    raise ValueError(f"{path}:{ln}: a face needs at least three vertices")
                idx = []
                for c in parts[1:]:
                    i = int(c.split("/")[0])
                    if i == 0:
                        raise ValueError(f"{path}:{ln}: OBJ vertex indices start at 1")
                    i = i - 1 if i > 0 else len(verts) + i
                    if not 0 <= i < len(verts):
                        raise ValueError(f"{path}:{ln}: vertex index {c} out of range (have {len(verts)} vertices)")
                    idx.append(i)
                faces.extend([idx[0], idx[k], idx[k + 1]] for k in range(1, len(idx) - 1))
    v = torch.tensor(np.asarray(verts, dtype=np.float32).reshape(-1, 3))
    f = torch.tensor(np.asarray(faces, dtype=np.int64).reshape(-1, 3))
    return v, f


def write_obj(path: str, vertices, faces, normals=None) -> None:
    """write_simple_obj's format: `v %f %f %f` per vertex, then `f %d %d %d` per face, 1-based.  With per-vertex normals
    [V,3]: `v %f %f %f`, then `vn %f %f %f` per vertex, then `f a//a b//b c//c` per face."""
    v = vertices.detach().cpu().numpy() if torch.is_tensor(vertices) else np.asarray(vertices)
    f = faces.detach().cpu().numpy() if torch.is_tensor(faces) else np.asarray(faces)
    if normals is not None:
        n = normals.detach().cpu().numpy() if torch.is_tensor(normals) else np.asarray(normals)
        if n.reshape(-1, 3).shape[0] != v.reshape(-1, 3).shape[0]:
            raise ValueError(f"write_obj: {n.reshape(-1, 3).shape[0]} normals for {v.reshape(-1, 3).shape[0]} vertices")
    with open(path, "w") as fp:
        for x in v.reshape(-1, 3):
            fp.write("v %f %f %f\n" % (x[0], x[1], x[2]))
        if normals is None:
            for t in f.reshape(-1, 3).astype(np.int64) + 1:
                fp.write("f %d %d %d\n" % (t[0], t[1], t[2]))
            return
        for x in n.reshape(-1, 3):
            fp.write("vn %f %f %f\n" % (x[0], x[1], x[2]))
        for t in f.reshape(-1, 3).astype(np.int64) + 1:
            fp.write("f %d//%d %d//%d %d//%d\n" % (t[0], t[0], t[1], t[1], t[2], t[2]))


def triangle_soup(triangles: torch.Tensor):
    """A pseudo-mesh [P,3,3] as the (vertices [3P,3], faces [P,3]) mesh the reference writes (three vertices per triangle,
    edit_pseudomesh_based_on_estimated_mesh.py:88-94), for write_obj."""
    P = triangles.shape[0]
    return triangles.reshape(P * 3, 3), torch.arange(P * 3, dtype=torch.int64).reshape(P, 3)
