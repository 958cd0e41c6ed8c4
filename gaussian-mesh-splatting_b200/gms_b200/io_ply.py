"""`point_cloud.ply` / `model_params.pt` IO without the `plyfile` dependency (SURVEY.md section 8f rank 4).

Layout = what the reference writes in GaussianModel._save_ply (scene/gaussian_model.py:177-216): one `vertex` element,
all properties float32, in the order  x y z nx ny nz f_dc_0..2 f_rest_0..(3*(M-1)-1) opacity scale_0..2 rot_0..3 ;
`f_dc` / `f_rest` are stored channel-major ([P,3,M-1] flattened) and transposed back to [P,M-1,3] on load
(scene/gaussian_model.py:224-262).  Mesh models add `model_params.pt` next to the PLY with `_alpha`, `_scale`, `vertices`,
`faces`, `triangles` (games/mesh_splatting/scene/gaussian_mesh_model.py:189-225).
Reads binary_little_endian (plyfile's default) and ascii PLY; writes binary_little_endian."""
from __future__ import annotations

import os
import pickle
import types
from typing import Dict, List, Tuple

import numpy as np
import torch

from .scenes import MeshGaussianParams

_TYPES = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1", "char": "i1",
          "int8": "i1", "short": "<i2", "int16": "<i2", "ushort": "<u2", "uint16": "<u2", "int": "<i4", "int32": "<i4",
          "uint": "<u4", "uint32": "<u4"}


def read_ply_vertices(path: str) -> Tuple[np.ndarray, List[str]]:
    """-> (structured array of the `vertex` element, property names)."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, count, props, in_vertex = None, 0, [], False
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: truncated PLY header")
            tok = line.decode("ascii", "replace").split()
            if not tok:
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    count = int(tok[2])
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError("list properties on the vertex element are not supported")
                props.append((tok[2], _TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        dtype = np.dtype(props)
        if fmt == "binary_little_endian":
            data = np.fromfile(f, dtype=dtype, count=count)
        elif fmt == "ascii":
            raw = np.loadtxt(f, max_rows=count, ndmin=2)
            data = np.empty(count, dtype=dtype)
            for i, (n, _) in enumerate(props):
                data[n] = raw[:, i]
        else:
            raise ValueError(f"{path}: unsupported PLY format {fmt}")
    if data.shape[0] != count:
        raise ValueError(f"{path}: expected {count} vertices, found {data.shape[0]}")
    return data, [n for n, _ in props]


_F_REST_COUNTS = {3 * ((d + 1) ** 2 - 1) for d in range(4)}      # 0, 9, 24, 45


def _sorted_cols(data, names, prefix):
    cols = sorted([n for n in names if n.startswith(prefix)], key=lambda x: int(x.split("_")[-1]))
    return np.stack([np.asarray(data[n], np.float32) for n in cols], axis=1) if cols else np.zeros((data.shape[0], 0), np.float32)


def load_gaussian_ply(path: str) -> Dict[str, torch.Tensor]:
    """-> dict(_xyz [P,3], _features_dc [P,1,3], _features_rest [P,M-1,3], _opacity [P,1], _scaling [P,S], _rotation [P,4])
    exactly as GaussianModel._load_ply builds them (scene/gaussian_model.py:224-262)."""
    data, names = read_ply_vertices(path)
    P = data.shape[0]
    xyz = np.stack([data["x"], data["y"], data["z"]], axis=1).astype(np.float32)
    fdc = _sorted_cols(data, names, "f_dc_")
    frest = _sorted_cols(data, names, "f_rest_")
    # the reference asserts 3 * ((max_sh_degree + 1)^2 - 1) f_rest properties (scene/gaussian_model.py:238-241); any other
    # count has no SH degree the rasterizer could evaluate
    if fdc.shape[1] != 3 or frest.shape[1] not in _F_REST_COUNTS:
        raise ValueError(f"{path}: {fdc.shape[1]} f_dc_* and {frest.shape[1]} f_rest_* properties; a Gaussian PLY has 3 f_dc_* and "
                         f"3 * ((d + 1)^2 - 1) f_rest_* for an SH degree d in 0..3, i.e. one of {sorted(_F_REST_COUNTS)}")
    fdc = fdc.reshape(P, 3, 1)
    frest = frest.reshape(P, 3, frest.shape[1] // 3)
    out = dict(_xyz=torch.tensor(xyz), _features_dc=torch.tensor(fdc).transpose(1, 2).contiguous(),
               _features_rest=torch.tensor(frest).transpose(1, 2).contiguous(),
               _opacity=torch.tensor(np.asarray(data["opacity"], np.float32)[:, None]),
               _scaling=torch.tensor(_sorted_cols(data, names, "scale_")), _rotation=torch.tensor(_sorted_cols(data, names, "rot")))
    return out


def save_gaussian_ply(path: str, xyz, features_dc, features_rest, opacity, scaling, rotation, eps_s0: float = 1e-8) -> None:
    """Writer with the reference's property order / channel-major SH layout (scene/gaussian_model.py:177-216).  A two-column
    `scaling` (flat Gaussians, gs_flat / gs_points) gets the constant log(eps_s0) column prepended, as _save_ply does (:196-199),
    so the file always carries scale_0..2."""
    t = lambda a: a.detach().cpu().float() if isinstance(a, torch.Tensor) else torch.as_tensor(a, dtype=torch.float32)
    xyz, fdc, frest, op, sc, rot = map(t, (xyz, features_dc, features_rest, opacity, scaling, rotation))
    P = xyz.shape[0]
    if sc.dim() == 2 and sc.shape[1] == 2:
        sc = torch.cat([torch.log(torch.ones(P, 1) * eps_s0), sc], dim=1)
    cols = [xyz, torch.zeros_like(xyz), fdc.transpose(1, 2).reshape(P, -1), frest.transpose(1, 2).reshape(P, -1), op.reshape(P, 1),
            sc.reshape(P, -1), rot.reshape(P, -1)]
    names = ["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(cols[2].shape[1])] + \
            [f"f_rest_{i}" for i in range(cols[3].shape[1])] + ["opacity"] + [f"scale_{i}" for i in range(cols[5].shape[1])] + \
            [f"rot_{i}" for i in range(cols[6].shape[1])]
    arr = np.ascontiguousarray(torch.cat(cols, dim=1).numpy().astype("<f4"))
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % P).encode())
        for n in names:
            f.write(f"property float {n}\n".encode())
        f.write(b"end_header\n")
        arr.tofile(f)


def load_mesh_model(ply_path: str) -> MeshGaussianParams:
    """point_cloud.ply + model_params.pt of a trained gs_mesh run -> raw parameters for MeshGaussianModel.from_params
    (GaussianMeshModel.load_ply, games/mesh_splatting/scene/gaussian_mesh_model.py:211-225)."""
    g = load_gaussian_ply(ply_path)
    params = torch.load(ply_path.replace("point_cloud.ply", "model_params.pt"), map_location="cpu", weights_only=False)
    d = lambda x: (x.detach() if isinstance(x, torch.Tensor) else torch.as_tensor(x)).cpu()
    verts = d(params["vertices"]).float()
    faces = d(params["faces"]).long()
    return MeshGaussianParams(verts, faces, d(params["_alpha"]).float(), d(params["_scale"]).float(), g["_features_dc"],
                              g["_features_rest"], g["_opacity"])


def save_mesh_model(ply_path: str, model) -> None:
    """Counterpart of GaussianMeshModel.save_ply (gaussian_mesh_model.py:189-209) for a gms_b200 MeshGaussianModel.
    model_params.pt holds what the reference's writer holds -- `_alpha`, `_scale`, `vertices` as nn.Parameters and
    `triangles`, `faces` as tensors, all ON THE MODEL'S DEVICE, plus the `point_cloud` key -- because the reference's
    load_ply (:211-225) uses them where they are (no .cuda()): a checkpoint written here loads in scripts/render.py."""
    model.update_alpha(); model.prepare_scaling_rot()
    save_gaussian_ply(ply_path, model._xyz, model._features_dc, model._features_rest, model._opacity, model._scaling, model._rotation,
                      getattr(model, "eps_s0", 1e-8))
    par = lambda t: torch.nn.Parameter(t.detach().clone().contiguous(), requires_grad=True)
    torch.save({"_alpha": par(model._alpha), "_scale": par(model._scale), "point_cloud": None,
                "triangles": model.triangles.detach().clone(), "vertices": par(model.vertices), "faces": model.faces.detach().clone()},
               ply_path.replace("point_cloud.ply", "model_params.pt"))


class _Opaque(tuple):
    """Stand-in for a class of the reference's own code pickled into model_params.pt (the `point_cloud` entries are
    games.multi_mesh_splatting.utils.graphics_utils.MultiMeshPointCloud named tuples): kept as a plain tuple of its fields."""

    def __new__(cls, *fields):
        return tuple.__new__(cls, fields)


class _Unpickler(pickle.Unpickler):
    def find_class(self, module, name):
        try:
            return super().find_class(module, name)
        except (ImportError, AttributeError):
            return _Opaque


_pickle_module = types.ModuleType("gms_b200_pickle")
_pickle_module.__dict__.update({k: getattr(pickle, k) for k in dir(pickle) if not k.startswith("__")})
_pickle_module.Unpickler = _Unpickler


def load_multi_mesh_model(ply_path: str) -> List[MeshGaussianParams]:
    """point_cloud.ply + model_params.pt of a trained gs_multi_mesh run -> one MeshGaussianParams per mesh, for
    MultiMeshGaussianModel.from_mesh_params (GaussianMultiMeshModel.load_ply, gaussian_multi_mesh_model.py:245-256).
    model_params.pt holds LISTS `_alpha` [F_i,K_i,3], `_scale` [F_i*K_i,1], `vertices` [V_i,3] and `faces` [F_i,3] (indices
    into mesh i's own vertices); the PLY's Gaussians are the meshes' in that order."""
    g = load_gaussian_ply(ply_path)
    params = torch.load(ply_path.replace("point_cloud.ply", "model_params.pt"), map_location="cpu", weights_only=False,
                        pickle_module=_pickle_module)
    d = lambda x: (x.detach() if isinstance(x, torch.Tensor) else torch.as_tensor(x)).cpu()
    out, g0 = [], 0
    for a, s, v, f in zip(params["_alpha"], params["_scale"], params["vertices"], params["faces"]):
        n = d(s).shape[0]
        out.append(MeshGaussianParams(d(v).float(), d(f).long(), d(a).float(), d(s).float(), g["_features_dc"][g0:g0 + n],
                                      g["_features_rest"][g0:g0 + n], g["_opacity"][g0:g0 + n]))
        g0 += n
    if g0 != g["_xyz"].shape[0]:
        raise ValueError(f"{ply_path}: {g['_xyz'].shape[0]} Gaussians in the PLY, {g0} in model_params.pt")
    return out


def save_multi_mesh_model(ply_path: str, model) -> None:
    """Counterpart of GaussianMultiMeshModel.save_ply (gaussian_multi_mesh_model.py:222-243) for a gms_b200
    MultiMeshGaussianModel (merged or segmented): point_cloud.ply, and model_params.pt with the reference's per-mesh LISTS
    `_alpha`, `_scale`, `vertices` (nn.Parameters) and `faces`, on the model's device, and `point_cloud` (empty: the
    reference's load_ply does not read it)."""
    model.update_alpha(); model.prepare_scaling_rot()
    save_gaussian_ply(ply_path, model._xyz, model._features_dc, model._features_rest, model._opacity, model._scaling, model._rotation,
                      getattr(model, "eps_s0", 1e-8))
    par = lambda t: torch.nn.Parameter(t.detach().clone().contiguous(), requires_grad=True)
    if model.segments is not None:
        views = model.mesh_views()
    else:
        views, f0, K = [], 0, model._alpha.shape[1]
        for F in model.mesh_face_counts:
            views.append((model.faces[f0:f0 + F], model._alpha[f0:f0 + F], model._scale[f0 * K:(f0 + F) * K]))
            f0 += F
    alphas, scales, verts, faces, v0 = [], [], [], [], 0
    for (f, a, s), nv in zip(views, model.mesh_vertex_counts):
        alphas.append(par(a)); scales.append(par(s)); verts.append(par(model.vertices[v0:v0 + nv])); faces.append((f - v0).detach().clone())
        v0 += nv
    torch.save({"_alpha": alphas, "_scale": scales, "point_cloud": [], "vertices": verts, "faces": faces},
               ply_path.replace("point_cloud.ply", "model_params.pt"))


# ---- point clouds (points3d.ply): scene/dataset_readers.py:107-130

_PCD_DTYPE = [("x", "f4"), ("y", "f4"), ("z", "f4"), ("nx", "f4"), ("ny", "f4"), ("nz", "f4"), ("red", "u1"), ("green", "u1"),
              ("blue", "u1")]


def point_cloud_elements(xyz, rgb) -> np.ndarray:
    """The `vertex` rows storePly builds (scene/dataset_readers.py:115-126): xyz and zero normals cast to f4, rgb cast to u1
    by numpy's float -> uint8 conversion, which truncates (127.9 -> 127)."""
    xyz, rgb = np.asarray(xyz), np.asarray(rgb)
    el = np.empty(xyz.shape[0], dtype=_PCD_DTYPE)
    for k, n in enumerate(("x", "y", "z")):
        el[n] = xyz[:, k]
    for n in ("nx", "ny", "nz"):
        el[n] = 0
    for k, n in enumerate(("red", "green", "blue")):
        el[n] = rgb[:, k]
    return el


def point_cloud_arrays(data) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """`vertex` rows -> (points [P,3], colors [P,3] = rgb / 255 in float64, normals [P,3]) as fetchPly returns them
    (scene/dataset_readers.py:107-113)."""
    points = np.vstack([data["x"], data["y"], data["z"]]).T
    colors = np.vstack([data["red"], data["green"], data["blue"]]).T / 255.0
    normals = np.vstack([data["nx"], data["ny"], data["nz"]]).T
    return points, colors, normals


def load_point_cloud(path: str) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """points3d.ply (COLMAP's converted cloud, or the random cloud of a NeRF-synthetic scene) -> (points [P,3] float32,
    colors [P,3] = rgb / 255, normals [P,3]): fetchPly (scene/dataset_readers.py:107-113).  Binary or ASCII."""
    data, _ = read_ply_vertices(path)
    return point_cloud_arrays(data)


def save_point_cloud(path: str, xyz, rgb) -> None:
    """storePly (scene/dataset_readers.py:115-130): binary little-endian `x y z nx ny nz` float (normals zero) and
    `red green blue` uchar, the colours truncated to bytes."""
    el = point_cloud_elements(xyz, rgb)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % el.shape[0]).encode())
        for n, t in _PCD_DTYPE:
            f.write(f"property {'float' if t == 'f4' else 'uchar'} {n}\n".encode())
        f.write(b"end_header\n")
        el.tofile(f)


# ---- gs_flame checkpoints: GaussianFlameModel.save_ply / load_ply (games/flame_splatting/scene/gaussian_flame_model.py:230-265)

FLAME_KEYS = ("_flame_shape", "_flame_exp", "_flame_pose", "_flame_neck_pose", "_flame_trans", "_vertices_enlargement", "faces",
              "alpha", "point_cloud")


def load_flame_model(ply_path: str) -> Dict[str, object]:
    """point_cloud.ply + flame_params.pt of a trained gs_flame run -> dict with load_gaussian_ply's tensors (_xyz,
    _features_dc, _features_rest, _opacity, _scaling, _rotation) and flame_params.pt's entries (FLAME_KEYS) as CPU tensors;
    `alpha` is the ACTIVATED weights [F,K,3] the reference stores, and there is no `_scales` (the reference does not save it).
    `point_cloud` is read through the unpickler that keeps classes of the reference's code as opaque tuples, so the reference
    need not be importable."""
    out = dict(load_gaussian_ply(ply_path))
    params = torch.load(ply_path.replace("point_cloud.ply", "flame_params.pt"), map_location="cpu", weights_only=False,
                        pickle_module=_pickle_module)
    d = lambda x: (x.detach() if isinstance(x, torch.Tensor) else torch.as_tensor(x)).cpu()
    for k in FLAME_KEYS[:-1]:
        out[k] = d(params[k]).long() if k == "faces" else d(params[k]).float()
    out["point_cloud"] = params.get("point_cloud")
    return out


def save_flame_model(ply_path: str, model, point_cloud=None) -> None:
    """Counterpart of GaussianFlameModel.save_ply for a gms_b200 FlameGaussianModel at its current parameters: point_cloud.ply
    (the expansion's _xyz, raw _scaling / _rotation, SH, opacity) and flame_params.pt with exactly the reference's keys --
    the six FLAME tensors as nn.Parameters, `faces`, the activated `alpha` and `point_cloud` (pickled as given) -- on the
    model's device, as the reference's writer leaves them."""
    from . import _lib, expansion
    verts = model.refresh_vertices()
    xyz, sc, rot, alpha, _ = expansion.expand(verts, model.faces, model._alpha.detach(), model._scales.detach(), model.eps_s0,
                                              activated=False, alpha_activation=_lib.ALPHA_SOFTMAX)
    f = model._features.detach()
    write_flame_checkpoint(ply_path, xyz, f[:, :1], f[:, 1:], model._opacity, sc, rot, {k: getattr(model, k) for k in FLAME_KEYS[:6]},
                           model.faces, alpha, point_cloud, model.eps_s0)


def write_flame_checkpoint(ply_path: str, xyz, features_dc, features_rest, opacity, scaling, rotation, flame: dict, faces, alpha,
                           point_cloud=None, eps_s0: float = 1e-8) -> None:
    """The two files of a gs_flame checkpoint from expanded tensors: point_cloud.ply (save_gaussian_ply) and flame_params.pt
    with the reference's keys -- the six FLAME tensors (`flame`) as nn.Parameters, `faces`, the activated `alpha`,
    `point_cloud` -- each where the caller holds it."""
    save_gaussian_ply(ply_path, xyz, features_dc, features_rest, opacity, scaling, rotation, eps_s0)
    par = lambda t: torch.nn.Parameter(torch.as_tensor(t).detach().clone().contiguous(), requires_grad=True)
    save = {k: par(flame[k]) for k in FLAME_KEYS[:6]}
    save.update(faces=torch.as_tensor(faces).detach().clone(), alpha=torch.as_tensor(alpha).detach().clone(), point_cloud=point_cloud)
    torch.save(save, ply_path.replace("point_cloud.ply", "flame_params.pt"))
