"""Fused mesh -> Gaussian expansion (autograd front end over gms_expand_forward / gms_expand_backward).

Replaces, per call, the ~45 ATen kernels (+ their autograd) of
  GaussianMeshModel.update_alpha / _calc_xyz        games/mesh_splatting/scene/gaussian_mesh_model.py:153-169, 86-101
  GaussianMeshModel.prepare_scaling_rot             games/mesh_splatting/scene/gaussian_mesh_model.py:103-151
  rot_to_quat_batch                                 utils/general_utils.py:43-96
  get_scaling / get_rotation activations            scene/gaussian_model.py:95-101
with ONE kernel forward and ONE kernel backward (vertex gradients scattered with float atomics).

Three entry points:
  expand(...)               everything from (vertices, faces, _alpha, _scale) in one launch  -- the fast path
  update_alpha_op(...)      alpha / triangles / xyz only        } the two-step protocol the reference's callers use
  prepare_scaling_rot_op()  _scaling / _rotation from triangles } (train.py:154-157, gaussian_animated_renderer:61-73)
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib

EPS_S0 = 1e-8   # gaussian_mesh_model.py:43


def _f32(t):
    t = t if (t.dtype == torch.float32 and t.is_contiguous()) else t.contiguous().float()
    return t.clone() if t.data_ptr() % 16 else t


def _stream(device):
    return torch.cuda.current_stream(device).cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _args(V, F, K, vertices, faces, triangles_in, alpha_raw, scale_raw, eps, alpha_activation=_lib.ALPHA_RELU, **outs):
    a = _lib.ExpandArgs()
    a.alpha_activation = int(alpha_activation)
    a.V, a.F, a.K = int(V), int(F), int(K)
    a.vertices, a.faces, a.triangles_in = _p(vertices), _p(faces), _p(triangles_in)
    a.alpha_raw, a.scale_raw, a.eps = _p(alpha_raw), _p(scale_raw), float(eps)
    for k in ("alpha", "triangles", "xyz", "scaling_log", "rotation_raw", "scaling_act", "rotation_act"):
        setattr(a, k, _p(outs.get(k)))
    return a


class _Expand(torch.autograd.Function):
    """vertices [V,3], faces [F,3] int64, _alpha [F,K,3], _scale [P,1] -> xyz, scaling, rotation (+alpha, triangles)."""

    @staticmethod
    def forward(ctx, vertices, faces, alpha_raw, scale_raw, eps, activated, alpha_activation):
        if not vertices.is_cuda:
            raise RuntimeError("gms_b200.expand: CUDA tensors required (no CPU path in the product)")
        L = _lib.lib()
        dev = vertices.device
        v, a, s = _f32(vertices.detach()), _f32(alpha_raw.detach()), _f32(scale_raw.detach())
        f = faces if (faces.dtype == torch.int64 and faces.is_contiguous()) else faces.long().contiguous()
        F, K = a.shape[0], a.shape[1]
        P = F * K
        e = lambda *sh: torch.empty(sh, dtype=torch.float32, device=dev)
        alpha, tri, xyz, sc, rot = e(F, K, 3), e(F, 3, 3), e(P, 3), e(P, 3), e(P, 4)
        outs = dict(alpha=alpha, triangles=tri, xyz=xyz)
        outs.update(dict(scaling_act=sc, rotation_act=rot) if activated else dict(scaling_log=sc, rotation_raw=rot))
        args = _args(v.shape[0], F, K, v, f, None, a, s, eps, alpha_activation, **outs)
        with torch.cuda.device(dev):
            _lib.check(L.gms_expand_forward(C.byref(args), _stream(dev)), "gms_expand_forward")
        ctx.save_for_backward(v, f, a, s)
        ctx.eps, ctx.activated, ctx.alpha_activation = float(eps), bool(activated), int(alpha_activation)
        ctx.mark_non_differentiable(alpha, tri)
        return xyz, sc, rot, alpha, tri

    @staticmethod
    def backward(ctx, g_xyz, g_sc, g_rot, _ga, _gt):
        L = _lib.lib()
        v, f, a, s = ctx.saved_tensors
        dev = v.device
        F, K = a.shape[0], a.shape[1]
        g = _lib.ExpandGrads()
        gx = None if g_xyz is None else _f32(g_xyz)
        gs = None if g_sc is None else _f32(g_sc)
        gr = None if g_rot is None else _f32(g_rot)
        g.dL_dxyz = _p(gx)
        if ctx.activated:
            g.dL_dscaling_act, g.dL_drotation_act = _p(gs), _p(gr)
        else:
            g.dL_dscaling_log, g.dL_drotation_raw = _p(gs), _p(gr)
        dv = torch.zeros_like(v)
        da = torch.empty_like(a)
        ds = torch.empty_like(s)
        g.dL_dvertices, g.dL_dalpha_raw, g.dL_dscale_raw = dv.data_ptr(), da.data_ptr(), ds.data_ptr()
        args = _args(v.shape[0], F, K, v, f, None, a, s, ctx.eps, ctx.alpha_activation)
        with torch.cuda.device(dev):
            _lib.check(L.gms_expand_backward(C.byref(args), C.byref(g), _stream(dev)), "gms_expand_backward")
        return dv, None, da, ds, None, None, None


def expand(vertices, faces, _alpha, _scale, eps: float = EPS_S0, activated: bool = True, alpha_activation: int = _lib.ALPHA_RELU):
    """One-launch expansion.  Returns (xyz [P,3], scaling [P,3], rotation [P,4], alpha [F,K,3], triangles [F,3,3]);
    scaling/rotation are ACTIVATED (exp / normalised) when `activated`, else the raw `_scaling` / `_rotation`.
    alpha_activation: _lib.ALPHA_RELU (gs_mesh: relu + 1e-8, normalised) or _lib.ALPHA_SOFTMAX (gs_flame: softmax)."""
    return _Expand.apply(vertices, faces, _alpha, _scale, eps, activated, alpha_activation)


class _UpdateAlpha(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vertices, faces, alpha_raw):
        if not vertices.is_cuda:
            raise RuntimeError("gms_b200.update_alpha: CUDA tensors required (no CPU path in the product)")
        L = _lib.lib()
        dev = vertices.device
        v, a = _f32(vertices.detach()), _f32(alpha_raw.detach())
        f = faces if (faces.dtype == torch.int64 and faces.is_contiguous()) else faces.long().contiguous()
        F, K = a.shape[0], a.shape[1]
        e = lambda *sh: torch.empty(sh, dtype=torch.float32, device=dev)
        alpha, tri, xyz = e(F, K, 3), e(F, 3, 3), e(F * K, 3)
        dummy_scale = torch.ones(F * K, 1, device=dev)
        args = _args(v.shape[0], F, K, v, f, None, a, dummy_scale, EPS_S0, alpha=alpha, triangles=tri, xyz=xyz)
        with torch.cuda.device(dev):
            _lib.check(L.gms_expand_forward(C.byref(args), _stream(dev)), "gms_expand_forward")
        ctx.save_for_backward(v, f, a, dummy_scale)
        return alpha, tri, xyz

    @staticmethod
    def backward(ctx, g_alpha, g_tri, g_xyz):
        L = _lib.lib()
        v, f, a, dummy = ctx.saved_tensors
        dev = v.device
        F, K = a.shape[0], a.shape[1]
        g = _lib.ExpandGrads()
        gx = torch.zeros(F * K, 3, device=dev) if g_xyz is None else _f32(g_xyz)
        dtri = torch.empty(F, 3, 3, device=dev)
        da = torch.empty_like(a)
        g.dL_dxyz, g.dL_dtriangles, g.dL_dalpha_raw = gx.data_ptr(), dtri.data_ptr(), da.data_ptr()
        args = _args(v.shape[0], F, K, v, f, None, a, dummy, EPS_S0)
        with torch.cuda.device(dev):
            _lib.check(L.gms_expand_backward(C.byref(args), C.byref(g), _stream(dev)), "gms_expand_backward")
        if g_tri is not None:
            dtri = dtri + g_tri
        dv = torch.zeros_like(v).index_add_(0, f.reshape(-1), dtri.reshape(-1, 3))
        if g_alpha is not None:
            # pc.alpha is consumed directly by renderer/gaussian_animated_renderer/__init__.py:61-64 and
            # flame_gaussian_renderer:60 (`torch.matmul(pc.alpha, triangles)`): backward of
            # alpha = r / sum(r), r = relu(_alpha) + 1e-8 (gaussian_mesh_model.py:166-167).  Rare path, ATen ops.
            r = torch.relu(a) + 1e-8
            ssum = r.sum(dim=-1, keepdim=True)
            alpha = r / ssum
            da = da + (g_alpha - (g_alpha * alpha).sum(dim=-1, keepdim=True)) / ssum * (a > 0).to(a.dtype)
        return dv, None, da


class _PrepareScalingRot(torch.autograd.Function):
    @staticmethod
    def forward(ctx, triangles, scale_raw, K, eps):
        if not triangles.is_cuda:
            raise RuntimeError("gms_b200.prepare_scaling_rot: CUDA tensors required (no CPU path in the product)")
        L = _lib.lib()
        dev = triangles.device
        t, s = _f32(triangles.detach()), _f32(scale_raw.detach())
        F = t.shape[0]
        P = F * K
        sc = torch.empty(P, 3, device=dev); rot = torch.empty(P, 4, device=dev)
        dummy_alpha = torch.ones(F, K, 3, device=dev)
        args = _args(0, F, K, None, None, t, dummy_alpha, s, eps, scaling_log=sc, rotation_raw=rot)
        with torch.cuda.device(dev):
            _lib.check(L.gms_expand_forward(C.byref(args), _stream(dev)), "gms_expand_forward")
        ctx.save_for_backward(t, s, dummy_alpha)
        ctx.K, ctx.eps = int(K), float(eps)
        return sc, rot

    @staticmethod
    def backward(ctx, g_sc, g_rot):
        L = _lib.lib()
        t, s, dummy_alpha = ctx.saved_tensors
        dev = t.device
        F, K = t.shape[0], ctx.K
        g = _lib.ExpandGrads()
        gs = None if g_sc is None else _f32(g_sc)
        gr = None if g_rot is None else _f32(g_rot)
        dtri = torch.empty(F, 3, 3, device=dev); ds = torch.empty_like(s)
        g.dL_dscaling_log, g.dL_drotation_raw = _p(gs), _p(gr)
        g.dL_dtriangles, g.dL_dscale_raw = dtri.data_ptr(), ds.data_ptr()
        args = _args(0, F, K, None, None, t, dummy_alpha, s, ctx.eps)
        with torch.cuda.device(dev):
            _lib.check(L.gms_expand_backward(C.byref(args), C.byref(g), _stream(dev)), "gms_expand_backward")
        return dtri, ds, None, None


def update_alpha_op(vertices, faces, _alpha):
    """-> (alpha [F,K,3], triangles [F,3,3], xyz [P,3]), all differentiable; gaussian_mesh_model.py:153-169."""
    return _UpdateAlpha.apply(vertices, faces, _alpha)


def prepare_scaling_rot_op(triangles, _scale, K: int, eps: float = EPS_S0):
    """-> (_scaling [P,3], _rotation [P,4]); gaussian_mesh_model.py:103-151."""
    return _PrepareScalingRot.apply(triangles, _scale, K, eps)


def patch_mesh_model(model):
    """Swap the fused ops into a reference-style GaussianMeshModel INSTANCE (duck-typed: needs vertices, faces,
    _alpha, _scale, eps_s0).  The reference's files stay untouched; train.py:154-157, scripts/render.py:43-48 and
    renderer/gaussian_animated_renderer/__init__.py:72-73 keep calling the same method names."""
    import types

    def update_alpha(self):
        self.alpha, self.triangles, self._xyz = update_alpha_op(self.vertices, self.faces, self._alpha)

    def prepare_scaling_rot(self):
        self._scaling, self._rotation = prepare_scaling_rot_op(self.triangles, self._scale, self.alpha.shape[1],
                                                               getattr(self, "eps_s0", EPS_S0))

    model.update_alpha = types.MethodType(update_alpha, model)
    model.prepare_scaling_rot = types.MethodType(prepare_scaling_rot, model)
    return model


def points_prepare_scaling_rot(triangles: torch.Tensor, eps: float = 1e-8, activated: bool = False):
    """gs_points pseudo-mesh: triangles [P,3,3] (one per Gaussian) -> (xyz [P,3] = triangles[:,0], scaling, rotation).
    activated=False: (_scaling [P,2], _rotation [P,4]) as PointsGaussianModel.prepare_scaling_rot stores them
    (games/flat_splatting/scene/points_gaussian_model.py:61-104); activated=True: (get_scaling [P,3], get_rotation [P,4]).
    Forward only (the reference calls it under no_grad, renderer/gaussian_points_animated_renderer/__init__.py:61-66)."""
    if not triangles.is_cuda:
        raise RuntimeError("points_prepare_scaling_rot: CUDA tensors required (no CPU path in the product)")
    t = _f32(triangles.detach())
    P, dev = t.shape[0], t.device
    xyz = torch.empty(P, 3, device=dev)
    sc = torch.empty(P, 3 if activated else 2, device=dev)
    rot = torch.empty(P, 4, device=dev)
    a = _lib.PointsArgs()
    a.P, a.triangles, a.eps, a.xyz = P, t.data_ptr(), float(eps), xyz.data_ptr()
    if activated:
        a.scaling_act, a.rotation_act = sc.data_ptr(), rot.data_ptr()
    else:
        a.scaling_log, a.rotation_raw = sc.data_ptr(), rot.data_ptr()
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().gms_points_expand_forward(C.byref(a), _stream(dev)), "gms_points_expand_forward")
    return xyz, sc, rot


def points_prepare_vertices(xyz: torch.Tensor, _scaling: torch.Tensor, _rotation: torch.Tensor) -> torch.Tensor:
    """gs_points: flat Gaussians -> pseudo-mesh triangles [P,3,3] (v1 = xyz; v2, v3 = xyz + exp(log-scale) * rotation axis,
    the longer arm first).  PointsGaussianModel.prepare_vertices, games/flat_splatting/scene/points_gaussian_model.py:28-59.
    `_scaling` is [P,2] or [P,3] (the last two columns are used, as get_scaling :106-109 does); `_rotation` is the raw
    (w,x,y,z) parameter (normalised inside, utils/general_utils.py:158-161).  Forward only."""
    if not xyz.is_cuda:
        raise RuntimeError("points_prepare_vertices: CUDA tensors required (no CPU path in the product)")
    x, sc, q = _f32(xyz.detach()), _f32(_scaling.detach()), _f32(_rotation.detach())
    P, dev = x.shape[0], x.device
    if sc.dim() != 2 or sc.shape[0] != P or sc.shape[1] not in (2, 3) or tuple(q.shape) != (P, 4) or tuple(x.shape) != (P, 3):
        raise ValueError("points_prepare_vertices: expected xyz [P,3], _scaling [P,2|3], _rotation [P,4]")
    tri = torch.empty(P, 3, 3, device=dev)
    a = _lib.PointsVerticesArgs()
    a.P, a.xyz, a.scaling_log, a.scaling_cols = P, x.data_ptr(), sc.data_ptr(), sc.shape[1]
    a.rotation_raw, a.triangles = q.data_ptr(), tri.data_ptr()
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().gms_points_prepare_vertices(C.byref(a), _stream(dev)), "gms_points_prepare_vertices")
    return tri


def patch_points_model(model):
    """Swap the fused kernels into a reference-style PointsGaussianModel instance: prepare_vertices() and
    prepare_scaling_rot(triangles=None, eps)."""
    import types

    def prepare_scaling_rot(self, triangles=None, eps=1e-8):
        tri = self.triangles if triangles is None else triangles
        _, self._scaling, self._rotation = points_prepare_scaling_rot(tri, eps, activated=False)

    def prepare_vertices(self):
        self.triangles = points_prepare_vertices(self._xyz, self._scaling, self._rotation)
        self.v1, self.v2, self.v3 = self.triangles.unbind(dim=1)

    model.prepare_scaling_rot = types.MethodType(prepare_scaling_rot, model)
    model.prepare_vertices = types.MethodType(prepare_vertices, model)
    return model


class PseudomeshBinding:
    """A pseudo-mesh bound to a driving mesh (bind_pseudomesh): `face` int32 [P] is each pseudo-triangle's face of that mesh,
    `coeffs` float32 [P,3,3] its three vertices in that face's (n, e1, e2) frame; `faces` int64 [F,3] and `V` fix the mesh
    every pose must share.  `n_degenerate` counts the faces of the rest pose that were never bound."""

    def __init__(self, face: torch.Tensor, coeffs: torch.Tensor, faces: torch.Tensor, V: int, n_degenerate: int):
        self.face, self.coeffs, self.faces, self.V, self.n_degenerate = face, coeffs, faces, int(V), int(n_degenerate)

    @property
    def P(self) -> int:
        return self.face.shape[0]

    def check_vertices(self, vertices: torch.Tensor) -> torch.Tensor:
        """A pose of the driving mesh as the kernels read it: contiguous float32 [V,3] on the binding's device."""
        if not torch.is_tensor(vertices) or tuple(vertices.shape) != (self.V, 3):
            raise ValueError(f"driving mesh pose: expected vertices [{self.V},3], got "
                             f"{tuple(vertices.shape) if torch.is_tensor(vertices) else type(vertices).__name__}")
        if vertices.device != self.face.device:
            raise ValueError(f"driving mesh pose: vertices must be on {self.face.device}")
        return _f32(vertices.detach())


def bind_pseudomesh(triangles: torch.Tensor, vertices: torch.Tensor, faces: torch.Tensor) -> PseudomeshBinding:
    """Bind every pseudo-triangle [P,3,3] to the nearest face (by centroid) of the mesh (vertices [V,3], faces [F,3]) and
    express its vertices in that face's frame: scripts/edit_pseudomesh_based_on_estimated_mesh.py:14-54 on the GPU, once per
    edit.  Degenerate faces (a zero edge or zero area) are never chosen; ValueError if the mesh has no other face.  Shapes,
    dtypes, the face-index range and finiteness are validated here, on the host, once."""
    if not (torch.is_tensor(triangles) and torch.is_tensor(vertices) and torch.is_tensor(faces)):
        raise TypeError("bind_pseudomesh: triangles, vertices and faces must be tensors")
    if not vertices.is_cuda:
        raise RuntimeError("bind_pseudomesh: CUDA tensors required (no CPU path in the product)")
    dev = vertices.device
    if triangles.device != dev or faces.device != dev:
        raise ValueError("bind_pseudomesh: triangles, vertices and faces must be on one device")
    if triangles.dim() != 3 or tuple(triangles.shape[1:]) != (3, 3) or vertices.dim() != 2 or vertices.shape[1] != 3 or \
            faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError("bind_pseudomesh: expected triangles [P,3,3], vertices [V,3], faces [F,3]")
    if not (triangles.is_floating_point() and vertices.is_floating_point()) or faces.is_floating_point() or faces.dtype == torch.bool:
        raise ValueError("bind_pseudomesh: triangles and vertices must be floating point, faces integer")
    P, V, F = triangles.shape[0], vertices.shape[0], faces.shape[0]
    if F < 1 or V < 1:
        raise ValueError("bind_pseudomesh: the mesh needs at least one face")
    if P >= 2 ** 31 or F >= 2 ** 31 or V >= 2 ** 31:
        raise ValueError("bind_pseudomesh: more than 2^31 - 1 triangles, faces or vertices")
    t, v, f = _f32(triangles.detach()), _f32(vertices.detach()), faces.detach().long().contiguous()
    if int(f.min()) < 0 or int(f.max()) >= V:
        raise ValueError(f"bind_pseudomesh: face indices must lie in [0, {V})")
    if not bool(torch.isfinite(t).all()) or not bool(torch.isfinite(v).all()):
        raise ValueError("bind_pseudomesh: triangles and vertices must be finite")
    face = torch.empty(P, dtype=torch.int32, device=dev)
    coeffs = torch.empty(P, 3, 3, dtype=torch.float32, device=dev)
    L = _lib.lib()
    scratch = torch.empty(int(L.gms_pseudomesh_bind_scratch_bytes(F)), dtype=torch.uint8, device=dev)
    nd = C.c_int32(0)
    a = _lib.PseudomeshBindArgs()
    a.P, a.triangles, a.V, a.F, a.vertices, a.faces = P, t.data_ptr(), V, F, v.data_ptr(), f.data_ptr()
    a.face, a.coeffs, a.n_degenerate = face.data_ptr(), coeffs.data_ptr(), C.pointer(nd)
    a.scratch, a.scratch_bytes = scratch.data_ptr(), scratch.numel()
    with torch.cuda.device(dev):
        rc = L.gms_pseudomesh_bind(C.byref(a), _stream(dev))
    if rc == _lib.GMS_E_ARG and nd.value >= F:
        raise ValueError(f"bind_pseudomesh: all {F} faces of the mesh are degenerate (zero edge or zero area)")
    _lib.check(rc, "gms_pseudomesh_bind")
    return PseudomeshBinding(face, coeffs, f, V, nd.value)


def repose_pseudomesh(binding: PseudomeshBinding, vertices: torch.Tensor) -> torch.Tensor:
    """The bound pseudo-mesh's triangles [P,3,3] in a pose (vertices [V,3]) of the driving mesh:
    scripts/edit_pseudomesh_based_on_estimated_mesh.py:58-82 (the `edited_triangles.pt` it saves).  A face degenerate in
    that pose gives non-finite triangles, as in the reference."""
    v = binding.check_vertices(vertices)
    P, dev = binding.P, v.device
    tri = torch.empty(P, 3, 3, dtype=torch.float32, device=dev)
    a = _lib.PseudomeshReposeArgs()
    a.P, a.face, a.coeffs, a.V, a.F = P, binding.face.data_ptr(), binding.coeffs.data_ptr(), binding.V, binding.faces.shape[0]
    a.vertices, a.faces, a.triangles = v.data_ptr(), binding.faces.data_ptr(), tri.data_ptr()
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().gms_pseudomesh_repose(C.byref(a), _stream(dev)), "gms_pseudomesh_repose")
    return tri
