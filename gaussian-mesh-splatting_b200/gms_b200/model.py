"""MeshGaussianModel -- the attribute surface renderer/*/__init__.py reads from a `pc`, backed by the fused ops.

Mirrors games/mesh_splatting/scene/gaussian_mesh_model.py (GaussianMeshModel) + the getters of
scene/gaussian_model.py:95-122 closely enough that the reference's `render(viewpoint_camera, pc, pipe, bg)`
(renderer/gaussian_renderer/__init__.py:25) and its animated variant run on it unchanged.  It exists so that
bench.py / tests do not need /root/reference at run time; a reference GaussianMeshModel instance can instead be
patched in place with expansion.patch_mesh_model().
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn

from . import _lib, expansion
from .scenes import SH_C0, MeshGaussianParams


class MeshGaussianModel:
    segments = None     # MultiMeshGaussianModel with a K per mesh: [(F_i, K_i), ...]; None: one K for every face
    alpha_activation = _lib.ALPHA_RELU      # barycentric weights from _alpha: relu + 1e-8, normalised (gaussian_mesh_model.py:166-167)

    def __init__(self, sh_degree: int = 3):
        self.active_sh_degree = 0
        self.max_sh_degree = sh_degree
        self.eps_s0 = expansion.EPS_S0
        self.vertices = self.faces = self._alpha = self._scale = None
        self._features = None
        self._opacity = None
        self.alpha = self.triangles = self._xyz = self._scaling = self._rotation = None
        self.optimizer = None

    @classmethod
    def from_params(cls, p: MeshGaussianParams, device="cuda", sh_degree: int = 3, active_sh_degree: int = 3,
                    packed_features: bool = False):
        """packed_features: keep SH coefficients in ONE [P,16,3] parameter (`_features`); `_features_dc` / `_features_rest`
        become views of it and get_features is zero-copy (the reference's torch.cat re-materialises 192 B/Gaussian
        every frame, scene/gaussian_model.py:107-111).  Needs FlatAdam for the DC / rest learning rates."""
        m = cls(sh_degree)
        m._adopt_params(p, device, active_sh_degree, packed_features)
        m.update_alpha()
        m.prepare_scaling_rot()
        return m

    def _adopt_params(self, p: MeshGaussianParams, device, active_sh_degree: int, packed_features: bool) -> None:
        self.active_sh_degree = active_sh_degree
        self.faces = p.faces.to(device)
        mk = lambda t: nn.Parameter(t.to(device).float().contiguous().requires_grad_(True))
        for k in ("vertices", "_alpha", "_scale", "_opacity"):
            setattr(self, k, mk(getattr(p, k)))
        if packed_features:
            self._features = mk(torch.cat((p._features_dc, p._features_rest), dim=1))
        else:
            self._features = None
            self._features_dc, self._features_rest = mk(p._features_dc), mk(p._features_rest)

    def frame_sizes(self):
        """(F, K, segments) as gms_frame_args / gms_render_args take them: K and no segments for one K per face; K = 0 and
        the host array of (F_i, K_i) for a segmented MultiMeshGaussianModel."""
        if self.segments is None:
            return self._alpha.shape[0], self._alpha.shape[1], None
        return self.faces.shape[0], 0, self._segment_array

    def __getattr__(self, name):   # only called when normal lookup fails: packed-mode views
        if name in ("_features_dc", "_features_rest") and self.__dict__.get("_features") is not None:
            f = self.__dict__["_features"]
            return f[:, :1] if name == "_features_dc" else f[:, 1:]
        raise AttributeError(name)

    # -- the two hooks train.py:154-157 calls every step
    def update_alpha(self):
        self.alpha, self.triangles, self._xyz = expansion.update_alpha_op(self.vertices, self.faces, self._alpha)

    def prepare_scaling_rot(self):
        self._scaling, self._rotation = expansion.prepare_scaling_rot_op(self.triangles, self._scale,
                                                                         self._alpha.shape[1], self.eps_s0)

    def expand_fused(self, activated: bool = True):
        """Fast path: one launch for E1-E4; returns (xyz, scaling, rotation) and refreshes alpha/triangles."""
        xyz, sc, rot, self.alpha, self.triangles = expansion.expand(self.vertices, self.faces, self._alpha, self._scale,
                                                                    self.eps_s0, activated)
        if not activated:
            self._xyz, self._scaling, self._rotation = xyz, sc, rot
        return xyz, sc, rot

    # -- getters (scene/gaussian_model.py:95-118)
    @property
    def get_xyz(self):
        return self._xyz

    @property
    def get_scaling(self):
        return torch.exp(self._scaling)

    @property
    def get_rotation(self):
        return torch.nn.functional.normalize(self._rotation)

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)

    @property
    def get_features(self):
        if self._features is not None:
            return self._features
        return torch.cat((self._features_dc, self._features_rest), dim=1)

    def oneupSHdegree(self):
        if self.active_sh_degree < self.max_sh_degree:
            self.active_sh_degree += 1

    def parameters(self):
        if self._features is not None:
            return [self.vertices, self._alpha, self._features, self._opacity, self._scale]
        return [self.vertices, self._alpha, self._features_dc, self._features_rest, self._opacity, self._scale]

    def training_setup(self, vertices_lr=0.0, alpha_lr=0.001, feature_lr=0.0025, opacity_lr=0.05, scaling_lr=0.005):
        """Adam groups of gaussian_mesh_model.py:171-183 (lrs: arguments_games/__init__.py:17-30)."""
        if self._features is not None:
            raise RuntimeError("packed features need gms_b200.optim.FlatAdam (per-coefficient learning rates)")
        groups = [{"params": [self.vertices], "lr": vertices_lr, "name": "vertices"},
                  {"params": [self._alpha], "lr": alpha_lr, "name": "alpha"},
                  {"params": [self._features_dc], "lr": feature_lr, "name": "f_dc"},
                  {"params": [self._features_rest], "lr": feature_lr / 20.0, "name": "f_rest"},
                  {"params": [self._opacity], "lr": opacity_lr, "name": "opacity"},
                  {"params": [self._scale], "lr": scaling_lr, "name": "scaling"}]
        self.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
        return self.optimizer


class PointsModel:
    """gs_points pseudo-mesh model for rendering: one triangle per Gaussian (PointsGaussianModel,
    games/flat_splatting/scene/points_gaussian_model.py, after prepare_vertices).  `triangles` [P,3,3] is what an editing
    script moves; the SH features stay packed in ONE [P,M,3] tensor (`_features`), so a frame reads them without the
    reference's per-frame torch.cat; `_opacity` [P,1] holds the logits.  The model carries no scaling / rotation: every
    frame derives them from the triangles (gms_points_render_frame)."""

    def __init__(self, triangles: torch.Tensor, features: torch.Tensor, opacity: torch.Tensor, active_sh_degree: int = 3,
                 eps_s0: float = 1e-8):
        P = triangles.shape[0]
        if tuple(triangles.shape) != (P, 3, 3) or features.dim() != 3 or tuple(features.shape[::2]) != (P, 3) or \
                tuple(opacity.shape) != (P, 1):
            raise ValueError("PointsModel: expected triangles [P,3,3], features [P,M,3], opacity [P,1]")
        f32 = lambda t: t.detach().float().contiguous()
        self.triangles, self._features, self._opacity = f32(triangles), f32(features), f32(opacity)
        self.max_sh_degree = int(round(features.shape[1] ** 0.5)) - 1
        self.active_sh_degree = min(int(active_sh_degree), self.max_sh_degree)
        self.eps_s0 = float(eps_s0)         # PointsGaussianModel.eps_s0 (:23), also prepare_scaling_rot's eps (:60)

    @classmethod
    def from_gaussians(cls, xyz, _scaling, _rotation, features_dc, features_rest, opacity, device="cuda",
                       active_sh_degree: int = 3) -> "PointsModel":
        """Flat Gaussians (raw parameters: `_scaling` [P,2|3] log-scales, `_rotation` [P,4]) -> their pseudo-mesh, as
        PointsGaussianModel.prepare_vertices builds it (expansion.points_prepare_vertices)."""
        d = lambda t: t.detach().to(device).float().contiguous()
        tri = expansion.points_prepare_vertices(d(xyz), d(_scaling), d(_rotation))
        return cls(tri, torch.cat((d(features_dc), d(features_rest)), dim=1), d(opacity), active_sh_degree)

    @classmethod
    def from_flat_checkpoint(cls, ply_path: str, device="cuda", active_sh_degree: int = 3) -> "PointsModel":
        """A trained gs_flat (or gs_points) point_cloud.ply -> its pseudo-mesh model: GaussianModel.load_ply, then
        prepare_vertices, as scripts/render_points_time_animated.py:53-56 loads a checkpoint.  The file's scale_0 column
        (log eps_s0 of a flat model) is ignored: the triangle spans the last two scales."""
        from . import io_ply
        g = io_ply.load_gaussian_ply(ply_path)
        return cls.from_gaussians(g["_xyz"], g["_scaling"], g["_rotation"], g["_features_dc"], g["_features_rest"], g["_opacity"],
                                  device, active_sh_degree)

    @property
    def get_features(self):
        return self._features

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)

    def bind_to_mesh(self, vertices: torch.Tensor, faces: torch.Tensor) -> "MeshBoundPointsModel":
        """Bind this pseudo-mesh to a driving mesh in its rest pose (vertices [V,3], faces [F,3]; e.g. io_obj.read_obj of the
        mesh an editor moves): every triangle tracks the nearest face, so any pose of that mesh re-poses the Gaussians
        (expansion.bind_pseudomesh; scripts/edit_pseudomesh_based_on_estimated_mesh.py)."""
        dev = self.triangles.device
        v = vertices.detach().to(dev).float().contiguous()
        binding = expansion.bind_pseudomesh(self.triangles, v, faces.detach().to(dev))
        return MeshBoundPointsModel(self, binding, v)


class MeshBoundPointsModel:
    """A gs_points pseudo-mesh driven by a mesh (PointsModel.bind_to_mesh): it shares the PointsModel's `_features` /
    `_opacity` and holds the binding and a current pose `vertices` [V,3] of the driving mesh, initially the rest pose.
    Setting `vertices` to an edited or animated pose moves the Gaussians; `triangles` materialises them
    (expansion.repose_pseudomesh), which MeshBoundPointsRenderer never needs."""

    def __init__(self, points: PointsModel, binding, vertices: torch.Tensor):
        self.points, self.binding = points, binding
        self.vertices = vertices

    @property
    def vertices(self) -> torch.Tensor:
        return self._vertices

    @vertices.setter
    def vertices(self, v: torch.Tensor) -> None:
        """A pose must be [V,3] on the binding's device (ValueError otherwise); it is kept as contiguous float32, without
        a copy when it already is one, so in-place edits of that tensor move the Gaussians too."""
        self._vertices = self.binding.check_vertices(v)

    @property
    def _features(self):
        return self.points._features

    @property
    def _opacity(self):
        return self.points._opacity

    @property
    def active_sh_degree(self):
        return self.points.active_sh_degree

    @property
    def eps_s0(self):
        return self.points.eps_s0

    @property
    def faces(self):
        return self.binding.faces

    @property
    def triangles(self) -> torch.Tensor:
        return expansion.repose_pseudomesh(self.binding, self.vertices)

    @property
    def get_features(self):
        return self._features

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)


class MultiMeshGaussianModel(MeshGaussianModel):
    """gs_multi_mesh: several meshes, one Gaussian set (games/multi_mesh_splatting/scene/gaussian_multi_mesh_model.py).

    The reference keeps per-mesh lists (vertices / faces / _alpha / _scale) and loops `expand -> torch.cat`
    (:99-119, :121-174, :176-199).  Per-face work is independent of which mesh a face belongs to, so the meshes are merged
    ONCE at construction (faces re-indexed into one vertex array).  When every mesh uses the same K the whole set runs
    through the single-mesh kernels: one launch instead of a loop, no concatenation.

    Meshes with different K (train.py --num_splats a b ...) give a SEGMENTED model: `_alpha` is [P,3] and `_scale` [P,1],
    mesh i's Gaussians being the rows [P_i, P_i + F_i*K_i), P_i = sum_{j<i} F_j*K_j -- the reference's torch.cat order -- and
    `segments` lists (F_i, K_i).  Every per-Gaussian tensor is flat, so FlatAdam and the native frames (gms_train_frame /
    gms_render_frame with gms_mesh_segment) see one Gaussian set; the expansion runs once per mesh.  A segmented model
    computes no expansion at construction: `alpha` (a per-mesh list), `triangles`, `_xyz`, `_scaling` and `_rotation` are
    set by update_alpha() / prepare_scaling_rot() or expand_fused(activated=False)."""

    @classmethod
    def from_mesh_params(cls, plist, device="cuda", sh_degree: int = 3, active_sh_degree: int = 3, packed_features: bool = False,
                         segmented: bool = False):
        """segmented=True keeps one segment per mesh even when every K is equal (what the per-mesh launches cost, against the
        merged model); meshes with different K are always segmented."""
        off, faces = 0, []
        for p in plist:
            faces.append(p.faces + off)
            off += p.vertices.shape[0]
        segmented = segmented or len({p._alpha.shape[1] for p in plist}) != 1
        alpha = [p._alpha.reshape(-1, 3) if segmented else p._alpha for p in plist]
        merged = MeshGaussianParams(torch.cat([p.vertices for p in plist]), torch.cat(faces), torch.cat(alpha),
                                    torch.cat([p._scale for p in plist]),
                                    torch.cat([p._features_dc for p in plist]), torch.cat([p._features_rest for p in plist]),
                                    torch.cat([p._opacity for p in plist]))
        if segmented:
            m = cls(sh_degree)
            m._adopt_params(merged, device, active_sh_degree, packed_features)
            m.segments = [(int(p._alpha.shape[0]), int(p._alpha.shape[1])) for p in plist]
            m._segment_array = _lib.mesh_segments(m.segments)
        else:
            m = cls.from_params(merged, device, sh_degree, active_sh_degree, packed_features)
        m.mesh_face_counts = [p.faces.shape[0] for p in plist]
        m.mesh_vertex_counts = [p.vertices.shape[0] for p in plist]
        return m

    def mesh_views(self):
        """Segmented model: per mesh, (faces [F_i,3] indexing the merged `vertices`, _alpha view [F_i,K_i,3], _scale view
        [F_i*K_i,1]).  Views of the current parameter storage (FlatAdam re-points it), so taken afresh on every call."""
        out, f0, g0 = [], 0, 0
        for F, K in self.segments:
            out.append((self.faces[f0:f0 + F], self._alpha[g0:g0 + F * K].view(F, K, 3), self._scale[g0:g0 + F * K]))
            f0, g0 = f0 + F, g0 + F * K
        return out

    def update_alpha(self):
        if self.segments is None:
            return super().update_alpha()
        outs = [expansion.update_alpha_op(self.vertices, f, a) for f, a, _ in self.mesh_views()]
        self.alpha = [o[0] for o in outs]       # per mesh [F_i,K_i,3], as the reference's list
        self.triangles, self._xyz = torch.cat([o[1] for o in outs]), torch.cat([o[2] for o in outs])

    def prepare_scaling_rot(self):
        if self.segments is None:
            return super().prepare_scaling_rot()
        outs, f0 = [], 0
        for (F, K), (_, _, s) in zip(self.segments, self.mesh_views()):
            outs.append(expansion.prepare_scaling_rot_op(self.triangles[f0:f0 + F], s, K, self.eps_s0))
            f0 += F
        self._scaling, self._rotation = torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])

    def expand_fused(self, activated: bool = True):
        """Segmented model: one fused launch per mesh, then cat (the autograd fast path of MeshTrainer(native=False))."""
        if self.segments is None:
            return super().expand_fused(activated)
        outs = [expansion.expand(self.vertices, f, a, s, self.eps_s0, activated) for f, a, s in self.mesh_views()]
        xyz, sc, rot = (torch.cat([o[i] for o in outs]) for i in range(3))
        self.alpha, self.triangles = [o[3] for o in outs], torch.cat([o[4] for o in outs])
        if not activated:
            self._xyz, self._scaling, self._rotation = xyz, sc, rot
        return xyz, sc, rot

    def training_setup(self, *args, **kwargs):
        if self.segments is not None:
            raise RuntimeError("a MultiMeshGaussianModel with a K per mesh trains with FlatAdam (MeshTrainer(fast=True)); "
                               "the reference's torch.optim.Adam op sequence (fast=False) is not supported for it")
        return super().training_setup(*args, **kwargs)

    @staticmethod
    def expand_per_mesh(vertices_list, faces_list, alpha_list, scale_list, eps: float = expansion.EPS_S0):
        """Reference-shaped path for heterogeneous K: per-mesh fused launch, then cat (-> xyz, _scaling, _rotation)."""
        outs = [expansion.expand(v, f, a, s, eps, activated=False)[:3] for v, f, a, s in
                zip(vertices_list, faces_list, alpha_list, scale_list)]
        return tuple(torch.cat([o[i] for o in outs]) for i in range(3))


class FreeGaussianModel:
    """gs / gs_flat: free Gaussians, raw parameters activated every frame (scene/gaussian_model.py:95-122;
    games/flat_splatting/scene/flat_gaussian_model.py:32-35 for gs_flat).  `_xyz` [P,3], `_scaling` [P,3] (gs) or [P,2]
    (gs_flat: the in-plane log-scales; get_scaling prepends the constant eps_s0), `_rotation` [P,4], `_opacity` [P,1] logits,
    and the SH coefficients packed in ONE [P,M,3] tensor `_features` (`_features_dc` / `_features_rest` are views of it)."""

    KINDS = ("gs", "gs_flat")
    NAMES = ("_xyz", "_scaling", "_rotation", "_opacity", "_features")

    def __init__(self, xyz, scaling, rotation, features, opacity, kind: str = "gs_flat", device="cuda", active_sh_degree: int = 0,
                 eps_s0: float = 1e-8):
        if kind not in self.KINDS:
            raise ValueError(f"FreeGaussianModel: kind must be one of {self.KINDS}; got {kind!r}")
        P = xyz.shape[0]
        cols = 3 if kind == "gs" else 2
        if scaling.dim() == 2 and scaling.shape[1] == 3 and cols == 2:
            scaling = scaling[:, 1:]            # a gs_flat checkpoint's scale_0 column is log(eps_s0): not a parameter
        if tuple(xyz.shape) != (P, 3) or tuple(scaling.shape) != (P, cols) or tuple(rotation.shape) != (P, 4) or \
                features.dim() != 3 or tuple(features.shape[::2]) != (P, 3) or tuple(opacity.shape) != (P, 1):
            raise ValueError(f"FreeGaussianModel({kind}): expected xyz [P,3], scaling [P,{cols}], rotation [P,4], features [P,M,3], "
                             "opacity [P,1]")
        self.kind, self.eps_s0 = kind, float(eps_s0)
        self.max_sh_degree = int(round(features.shape[1] ** 0.5)) - 1
        self.active_sh_degree = min(int(active_sh_degree), self.max_sh_degree)
        mk = lambda t: nn.Parameter(t.detach().to(device).float().contiguous().requires_grad_(True))
        self._xyz, self._scaling, self._rotation, self._features, self._opacity = map(mk, (xyz, scaling, rotation, features, opacity))

    @classmethod
    def from_checkpoint(cls, ply_path: str, kind: str = "gs_flat", device="cuda", active_sh_degree: int = 3) -> "FreeGaussianModel":
        """A point_cloud.ply the reference (or save()) wrote: GaussianModel.load_ply (scene/gaussian_model.py:224-262)."""
        from . import io_ply
        g = io_ply.load_gaussian_ply(ply_path)
        return cls(g["_xyz"], g["_scaling"], g["_rotation"], torch.cat((g["_features_dc"], g["_features_rest"]), dim=1), g["_opacity"],
                   kind, device, active_sh_degree)

    @classmethod
    def from_point_cloud(cls, points, colors, kind: str = "gs_flat", sh_degree: int = 3, device="cuda") -> "FreeGaussianModel":
        """create_from_pcd (scene/gaussian_model.py:124-147; flat_gaussian_model.py:37-60 for gs_flat): points [P,3] and
        colors [P,3] in [0,1] (io_ply.load_point_cloud, scenes.random_point_cloud) ->
          _xyz = points.float(); DC = RGB2SH(colors), rest 0; _rotation = (1,0,0,0); _opacity = inverse_sigmoid(0.1);
          _scaling = log(sqrt(clamp_min(dist2, 1e-7))) over 3 columns (gs) or 2 (gs_flat), dist2 = knn.mean_dist2(_xyz);
          active_sh_degree = 0.
        RGB2SH is evaluated in float32 on the host, where the colours arrive; the scale and opacity maths is ATen on the device."""
        from . import knn
        xyz = torch.as_tensor(points).detach().float().to(device)
        rgb = torch.as_tensor(colors).detach().cpu().float()
        if xyz.dim() != 2 or xyz.shape[1] != 3 or tuple(rgb.shape) != tuple(xyz.shape):
            raise ValueError("from_point_cloud: expected points [P,3] and colors [P,3]")
        P, M = xyz.shape[0], (int(sh_degree) + 1) ** 2
        features = torch.zeros(P, M, 3)
        features[:, 0] = (rgb - 0.5) / SH_C0
        dist2 = torch.clamp_min(knn.mean_dist2(xyz), 0.0000001)
        scaling = torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3 if kind == "gs" else 2)
        rotation = torch.zeros(P, 4, device=xyz.device)
        rotation[:, 0] = 1
        x = 0.1 * torch.ones(P, 1, dtype=torch.float, device=xyz.device)
        opacity = torch.log(x / (1 - x))
        return cls(xyz, scaling, rotation, features, opacity, kind, device, active_sh_degree=0)

    def save(self, ply_path: str) -> None:
        """The reference's point_cloud.ply (GaussianModel.save_ply; gs_flat gets the log(eps_s0) scale_0 column)."""
        from . import io_ply
        io_ply.save_gaussian_ply(ply_path, self._xyz, self._features_dc, self._features_rest, self._opacity, self._scaling,
                                 self._rotation, self.eps_s0)

    @property
    def P(self) -> int:
        return self._xyz.shape[0]

    @property
    def scale_cols(self) -> int:
        return self._scaling.shape[1]

    @property
    def _features_dc(self):
        return self._features[:, :1]

    @property
    def _features_rest(self):
        return self._features[:, 1:]

    @property
    def get_xyz(self):
        return self._xyz

    @property
    def get_scaling(self):
        s = torch.exp(self._scaling)
        if self.kind == "gs":
            return s
        return torch.cat([torch.full((s.shape[0], 1), self.eps_s0, dtype=s.dtype, device=s.device), s], dim=1)

    @property
    def get_rotation(self):
        return torch.nn.functional.normalize(self._rotation)

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)

    @property
    def get_features(self):
        return self._features

    def oneupSHdegree(self):
        if self.active_sh_degree < self.max_sh_degree:
            self.active_sh_degree += 1

    def parameters(self):
        return [getattr(self, n) for n in self.NAMES]


# ---------------------------------------------------------------------------------------------- gs_flame (FLAME-driven mesh)

FLAME_ENLARGEMENT = 8.35        # FlameConfig.vertices_enlargement (games/flame_splatting/FLAME/config.py:28)


def flame_transform_vertices(vertices: torch.Tensor, enlargement) -> torch.Tensor:
    """transform_vertices_function (games/flame_splatting/scene/dataset_readers.py:40-45) out of place: the driver's
    [1,V,3] (or [V,3]) vertices as (x, -z, y) times `enlargement` ([V,3] or a scalar), element for element the same
    rounding as the reference's in-place version (a negation is exact)."""
    v = vertices.reshape(-1, 3)
    sign = torch.tensor([1.0, -1.0, 1.0], dtype=v.dtype, device=v.device)
    return v[:, [0, 2, 1]] * sign * enlargement


class FlameGaussianModel:
    """gs_flame: K Gaussians on every face of a FLAME head mesh (GaussianFlameModel,
    games/flame_splatting/scene/gaussian_flame_model.py).  The Gaussian parameters are `_alpha` [F,K,3] (barycentric logits,
    weighted through a softmax), `_scales` [P,1], the packed SH `_features` [P,M,3] and `_opacity` [P,1]; the mesh is the
    output of a caller-supplied FLAME `driver` with the reference's FLAME.forward signature
        driver(shape_params, expression_params, pose_params, neck_pose, transl) -> (vertices [1,V,3], landmarks)
    at the model's six FLAME tensors, through flame_transform_vertices.  The library never looks inside the driver: it runs
    in ATen with autograd, and the frame's vertex gradient is pushed back through it (FlameTrainer).

    `vertices` [V,3] is the pose the native frames and NativeRenderer read; refresh_vertices() sets it from the current
    parameters."""
    alpha_activation = _lib.ALPHA_SOFTMAX
    segments = None
    FLAME_NAMES = ("_flame_shape", "_flame_exp", "_flame_pose", "_flame_neck_pose", "_flame_trans", "_vertices_enlargement")

    def __init__(self, driver, faces: torch.Tensor, _alpha: torch.Tensor, _scales: torch.Tensor, features: torch.Tensor,
                 opacity: torch.Tensor, flame: dict, active_sh_degree: int = 0, eps_s0: float = expansion.EPS_S0):
        F, K = _alpha.shape[:2]
        P = F * K
        if _alpha.dim() != 3 or _alpha.shape[2] != 3 or tuple(_scales.shape) != (P, 1) or features.dim() != 3 or \
                tuple(features.shape[::2]) != (P, 3) or tuple(opacity.shape) != (P, 1) or tuple(faces.shape) != (F, 3):
            raise ValueError("FlameGaussianModel: expected faces [F,3], _alpha [F,K,3], _scales / _opacity [F*K,1], features [F*K,M,3]")
        dev = _alpha.device
        mk = lambda t: nn.Parameter(t.detach().to(dev).float().contiguous().requires_grad_(True))
        self.driver = driver
        self.faces = faces.detach().to(dev).long().contiguous()
        self._alpha, self._scales, self._features, self._opacity = mk(_alpha), mk(_scales), mk(features), mk(opacity)
        for n in self.FLAME_NAMES:
            setattr(self, n, mk(flame[n]))
        self.max_sh_degree = int(round(features.shape[1] ** 0.5)) - 1
        self.active_sh_degree = min(int(active_sh_degree), self.max_sh_degree)
        self.eps_s0 = float(eps_s0)
        V = self._vertices_enlargement.shape[0]
        self.vertices = torch.zeros(V, 3, dtype=torch.float32, device=dev)
        self.vertices.grad = torch.zeros_like(self.vertices)     # the frames' dL/dvertices (accumulated with atomics)
        self.refresh_vertices()

    @classmethod
    def create(cls, driver, faces: torch.Tensor, K: int = 100, sh_degree: int = 3, seed: int = 0, device="cuda",
               n_shape: int = 100, n_exp: int = 50) -> "FlameGaussianModel":
        """A new model as readNerfSyntheticFlameInfo + create_from_pcd build it (games/flame_splatting/scene/
        dataset_readers.py:48-120, gaussian_flame_model.py:58-105): FLAME parameters zero, enlargement 8.35 per vertex
        coordinate, `_alpha` ~ U[0,1) [F,K,3], colours np.random.random / 255 through SH2RGB / RGB2SH, `_scales` 1 and
        opacity inverse_sigmoid(0.1).  The draws come from torch / numpy generators seeded with `seed`."""
        dev = torch.device(device)
        zeros = lambda n: torch.zeros(1, n, dtype=torch.float32, device=dev)
        flame = dict(_flame_shape=zeros(n_shape), _flame_exp=zeros(n_exp), _flame_pose=zeros(6), _flame_neck_pose=zeros(3),
                     _flame_trans=zeros(3))
        with torch.no_grad():
            v0, _ = driver(shape_params=flame["_flame_shape"], expression_params=flame["_flame_exp"], pose_params=flame["_flame_pose"],
                           neck_pose=flame["_flame_neck_pose"], transl=flame["_flame_trans"])
        V = v0.reshape(-1, 3).shape[0]
        flame["_vertices_enlargement"] = FLAME_ENLARGEMENT * torch.ones(V, 3, dtype=torch.float32, device=dev)
        F = faces.shape[0]
        P = F * K
        g = torch.Generator().manual_seed(int(seed))
        alpha = torch.rand(F, K, 3, generator=g)
        shs = np.random.RandomState(seed).random_sample((P, 3)) / 255.0
        colors = shs * SH_C0 + 0.5                                        # SH2RGB
        fused = (torch.tensor(colors).float() - 0.5) / SH_C0              # RGB2SH
        M = (sh_degree + 1) ** 2
        features = torch.zeros(P, M, 3)
        features[:, 0, :] = fused
        opacity = torch.full((P, 1), 0.1)
        opacity = torch.log(opacity / (1 - opacity))                      # inverse_sigmoid
        return cls(driver, faces.to(dev), alpha.to(dev), torch.ones(P, 1, device=dev), features.to(dev), opacity.to(dev), flame)

    # -- the mesh
    def driver_vertices(self) -> torch.Tensor:
        """update_alpha's mesh (gaussian_flame_model.py:196-205): the driver at the FLAME parameters, transformed; [V,3] with
        autograd to the six FLAME tensors."""
        v, _ = self.driver(shape_params=self._flame_shape, expression_params=self._flame_exp, pose_params=self._flame_pose,
                           neck_pose=self._flame_neck_pose, transl=self._flame_trans)
        return flame_transform_vertices(v, self._vertices_enlargement)

    def refresh_vertices(self) -> torch.Tensor:
        with torch.no_grad():
            self.vertices.copy_(self.driver_vertices())
        return self.vertices

    # -- what the native frames read (MeshGaussianModel's surface)
    @property
    def _scale(self):
        return self._scales

    @property
    def P(self) -> int:
        return self._scales.shape[0]

    def frame_sizes(self):
        return self._alpha.shape[0], self._alpha.shape[1], None

    @property
    def alpha(self) -> torch.Tensor:
        """The activated barycentric weights softmax(_alpha) [F,K,3] (update_alpha_func, gaussian_flame_model.py:195)."""
        return expansion.expand(self.vertices, self.faces, self._alpha.detach(), self._scales.detach(), self.eps_s0,
                                alpha_activation=_lib.ALPHA_SOFTMAX)[3]

    @property
    def get_features(self):
        return self._features

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)

    def oneupSHdegree(self):
        if self.active_sh_degree < self.max_sh_degree:
            self.active_sh_degree += 1

    def parameters(self):
        return [getattr(self, n) for n in self.FLAME_NAMES] + [self._alpha, self._features, self._opacity, self._scales]


class FlameCheckpoint:
    """A trained gs_flame checkpoint as scripts/render_flame.py renders it (io_ply.load_flame_model): the activated weights
    `alpha` [F,K,3], `faces`, the raw `_scaling` [P,3] / `_rotation` [P,4] rows, packed `_features` [P,M,3], `_opacity`
    and the six FLAME tensors.  `vertices` [V,3] is the pose FlameRenderer draws when render() is given none (None until
    set, e.g. to flame_transform_vertices(driver(...), ckpt._vertices_enlargement))."""

    def __init__(self, ckpt: dict, device="cuda", active_sh_degree: int = 3):
        d = lambda t: torch.as_tensor(t).detach().to(device).float().contiguous()
        self.faces = torch.as_tensor(ckpt["faces"]).to(device).long().contiguous()
        self.alpha, self._scaling, self._rotation, self._opacity = (d(ckpt[k]) for k in ("alpha", "_scaling", "_rotation", "_opacity"))
        self._features = torch.cat((d(ckpt["_features_dc"]), d(ckpt["_features_rest"])), dim=1).contiguous()
        for n in FlameGaussianModel.FLAME_NAMES:
            setattr(self, n, d(ckpt[n]))
        self.max_sh_degree = int(round(self._features.shape[1] ** 0.5)) - 1
        self.active_sh_degree = min(int(active_sh_degree), self.max_sh_degree)
        self.vertices = None
        F, K = self.alpha.shape[:2]
        P = F * K
        if tuple(self._scaling.shape) != (P, 3) or tuple(self._rotation.shape) != (P, 4) or self._features.shape[0] != P or \
                tuple(self._opacity.shape) != (P, 1):
            raise ValueError(f"FlameCheckpoint: alpha [{F},{K},3] needs {P} Gaussian rows")

    @classmethod
    def load(cls, ply_path: str, device="cuda", active_sh_degree: int = 3) -> "FlameCheckpoint":
        from . import io_ply
        return cls(io_ply.load_flame_model(ply_path), device, active_sh_degree)

    @property
    def P(self) -> int:
        return self._opacity.shape[0]

    def driver_vertices(self, driver, **overrides) -> torch.Tensor:
        """The pose render_flame.py draws (:23-33): the driver at the checkpoint's FLAME parameters, any of them replaced by
        `overrides` (shape_params, expression_params, pose_params, neck_pose, transl -- e.g. the --animated expressions)."""
        kw = dict(shape_params=self._flame_shape, expression_params=self._flame_exp, pose_params=self._flame_pose,
                  neck_pose=self._flame_neck_pose, transl=self._flame_trans)
        kw.update(overrides)
        with torch.no_grad():
            v, _ = driver(**kw)
            return flame_transform_vertices(v, self._vertices_enlargement).contiguous()
