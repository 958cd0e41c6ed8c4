"""FLAME's vertex model on the GPU: linear blend skinning forward and backward as the library's own kernels
(gms_flame_lbs_forward / gms_flame_lbs_backward, csrc/gms_flame.cuh).

NativeFlame is a drop-in for the reference's FLAME module (games/flame_splatting/FLAME/FLAME.py) as a gs_flame driver:
called with FLAME.forward's arguments it returns (vertices [1,V,3], None) -- no landmarks -- and the vertices carry autograd
to the parameters through the backward kernel.  FlameTrainer skips autograd altogether when the model's driver is a
NativeFlame: it runs the forward straight into model.vertices and the backward straight into the optimizer's gradient
slots (NativeFlame.bind).

Three ways to build one:
  NativeFlame.from_model_file(path)        FLAME's model pickle (generic_model.pkl, flame2023.pkl), read without smplx,
                                           chumpy or scipy;
  NativeFlame.from_checkpoint(point_cloud) the `point_cloud` entry of io_ply.load_flame_model: the reference's pickled
                                           FLAMEPointCloud (its FLAME module's buffers), or the dict to_point_cloud() gives;
  NativeFlame(buffers...)                  tensors, e.g. the buffers of the reference's module."""
from __future__ import annotations

import ctypes as C
import pickle
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib

N_SHAPE_TOTAL, N_EXP_TOTAL = 300, 100      # FLAME's shape / expression basis: shapedirs [V,3,400]
PARENTS = (-1, 0, 1, 1, 1)                 # global -> neck -> (jaw, left eye, right eye)


class NativeFlame:
    def __init__(self, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, faces=None, n_shape: int = 100,
                 n_exp: int = 50, device="cuda"):
        """v_template [V,3], shapedirs [V,3,S], posedirs [36,3V], J_regressor [5,V], parents [5], lbs_weights [V,5] as the
        buffers of FLAME.__init__ (FLAME.py:93-121); faces [F,3].  S = 400 is FLAME's basis: columns [0, n_shape) and
        [300, 300 + n_exp) are the active ones.  S = n_shape + n_exp is a basis already packed to them, in that order."""
        t = lambda x: torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).detach()
        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())     # compared against the parameters' devices
        v_template, shapedirs, posedirs, J_regressor, lbs_weights = map(t, (v_template, shapedirs, posedirs, J_regressor, lbs_weights))
        n_shape, n_exp = int(n_shape), int(n_exp)
        if not (0 <= n_shape <= N_SHAPE_TOTAL and 0 <= n_exp <= N_EXP_TOTAL):
            raise ValueError(f"NativeFlame: need 0 <= n_shape <= 300 and 0 <= n_exp <= 100; got {n_shape}, {n_exp}")
        V = v_template.shape[0]
        if V < 1 or tuple(v_template.shape) != (V, 3) or shapedirs.dim() != 3 or tuple(shapedirs.shape[:2]) != (V, 3) or \
                tuple(posedirs.shape) != (36, 3 * V) or tuple(J_regressor.shape) != (_lib.FLAME_JOINTS, V) or \
                tuple(lbs_weights.shape) != (V, _lib.FLAME_JOINTS):
            raise ValueError("NativeFlame: expected v_template [V,3], shapedirs [V,3,S], posedirs [36,3V], J_regressor [5,V], "
                             f"lbs_weights [V,5]; got {[tuple(x.shape) for x in (v_template, shapedirs, posedirs, J_regressor, lbs_weights)]}")
        S, B = shapedirs.shape[2], n_shape + n_exp
        if S == N_SHAPE_TOTAL + N_EXP_TOTAL:
            cols = list(range(n_shape)) + list(range(N_SHAPE_TOTAL, N_SHAPE_TOTAL + n_exp))
        elif S == B:
            cols = list(range(B))
        else:
            raise ValueError(f"NativeFlame: shapedirs has {S} columns; expected 400 (FLAME's basis) or n_shape + n_exp = {B}")
        self.parents = tuple(int(p) for p in t(parents).reshape(-1).tolist())
        if len(self.parents) != _lib.FLAME_JOINTS or self.parents[0] != -1 or \
                any(not 0 <= p < j for j, p in enumerate(self.parents) if j):
            raise ValueError(f"NativeFlame: parents must be 5 joints with parents[0] = -1 and 0 <= parents[j] < j; got {self.parents}")
        self.V, self.n_shape, self.n_exp = V, n_shape, n_exp
        self.device = dev
        f32 = lambda x: x.to(dev, torch.float32).contiguous()
        self.v_template = f32(v_template)
        self.shapedirs = f32(shapedirs[:, :, cols].permute(2, 0, 1).reshape(B, 3 * V))     # packed [B,3V]
        self.posedirs = f32(posedirs)
        self.J_regressor = f32(J_regressor)
        self.lbs_weights = f32(lbs_weights)
        self.faces = None if faces is None else np.asarray(t(faces).numpy())
        self.faces_tensor = None if faces is None else torch.as_tensor(self.faces.astype(np.int64), device=dev)
        self._ones = torch.ones(V, 3, dtype=torch.float32, device=dev)
        self._ws_bytes = int(_lib.lib().gms_flame_lbs_workspace_bytes(V))

    # -- construction
    @classmethod
    def from_model_file(cls, path: str, n_shape: int = 100, n_exp: int = 50, device="cuda") -> "NativeFlame":
        """FLAME's model pickle -> the buffers exactly as FLAME.__init__ casts and reshapes them (FLAME.py:93-121): keys
        v_template, f, shapedirs, posedirs, J_regressor (dense, or a pickled scipy sparse matrix), kintree_table, weights;
        chumpy arrays are read from their pickled state."""
        with open(path, "rb") as fh:
            d = _ModelUnpickler(fh, encoding="latin1").load()
        if not isinstance(d, dict):
            raise ValueError(f"{path}: not a FLAME model file (a pickled dict)")
        arr = {}
        for k in ("v_template", "f", "shapedirs", "posedirs", "J_regressor", "kintree_table", "weights"):
            if k not in d:
                raise ValueError(f"{path}: FLAME model file has no {k!r}")
            arr[k] = _to_array(d[k], k)
        f32 = lambda a: torch.tensor(np.array(a, dtype=np.float32))         # smplx.utils.to_np / to_tensor
        posedirs = np.reshape(arr["posedirs"], [-1, arr["posedirs"].shape[-1]]).T
        parents = f32(arr["kintree_table"][0]).long()
        parents[0] = -1
        return cls(f32(arr["v_template"]), f32(arr["shapedirs"]), f32(posedirs), f32(arr["J_regressor"]), parents,
                   f32(arr["weights"]), arr["f"], n_shape, n_exp, device)

    @classmethod
    def from_checkpoint(cls, point_cloud, device="cuda") -> "NativeFlame":
        """The `point_cloud` entry of io_ply.load_flame_model: the reference's FLAMEPointCloud, whose `flame_model` (field 6)
        is its FLAME module -- v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights and faces_tensor are its
        buffers, n_shape / n_exp follow from its zero-padding parameters -- or the dict to_point_cloud() returns."""
        if isinstance(point_cloud, dict):
            return cls(device=device, **point_cloud)
        if not isinstance(point_cloud, tuple) or len(point_cloud) < 7:
            raise ValueError("NativeFlame.from_checkpoint: expected a FLAMEPointCloud or a to_point_cloud() dict")
        state = vars(point_cloud[6])
        buf, par = state.get("_buffers"), state.get("_parameters")
        if buf is None or par is None or "shape_betas" not in par:
            raise ValueError("NativeFlame.from_checkpoint: the checkpoint's flame_model is not a FLAME module")
        if not state.get("use_3D_translation", True):
            raise ValueError("NativeFlame.from_checkpoint: FLAME without use_3D_translation is not supported")
        n_shape = N_SHAPE_TOTAL - par["shape_betas"].shape[1]
        n_exp = N_EXP_TOTAL - par["expression_betas"].shape[1]
        return cls(buf["v_template"], buf["shapedirs"], buf["posedirs"], buf["J_regressor"], buf["parents"], buf["lbs_weights"],
                   buf["faces_tensor"], n_shape, n_exp, device)

    def to_point_cloud(self) -> dict:
        """The buffers as CPU tensors (shapedirs packed to the active columns, [V,3,n_shape + n_exp]): pass it to
        io_ply.save_flame_model(..., point_cloud=...) and from_checkpoint rebuilds this model from the checkpoint alone."""
        B = self.n_shape + self.n_exp
        c = lambda x: x.detach().cpu().clone()
        return dict(v_template=c(self.v_template), shapedirs=c(self.shapedirs.reshape(B, self.V, 3).permute(1, 2, 0).contiguous()),
                    posedirs=c(self.posedirs), J_regressor=c(self.J_regressor), parents=torch.tensor(self.parents, dtype=torch.long),
                    lbs_weights=c(self.lbs_weights), faces=None if self.faces is None else torch.as_tensor(self.faces.astype(np.int64)),
                    n_shape=self.n_shape, n_exp=self.n_exp)

    # -- the kernels
    def _args(self, shape, expression, pose, neck_pose, transl, enlargement, workspace, vertices=None, vertices_grad=None,
              grads: Optional[Sequence[torch.Tensor]] = None) -> "_lib.FlameLbsArgs":
        p = lambda x: 0 if x is None else x.data_ptr()
        a = _lib.FlameLbsArgs()
        a.V, a.n_shape, a.n_exp, a.n_joints = self.V, self.n_shape, self.n_exp, _lib.FLAME_JOINTS
        for j, q in enumerate(self.parents):
            a.parents[j] = q
        a.v_template, a.shapedirs, a.posedirs = p(self.v_template), p(self.shapedirs), p(self.posedirs)
        a.J_regressor, a.lbs_weights = p(self.J_regressor), p(self.lbs_weights)
        a.shape, a.expression, a.pose, a.neck_pose, a.transl, a.enlargement = map(p, (shape, expression, pose, neck_pose, transl, enlargement))
        a.vertices, a.vertices_grad = p(vertices), p(vertices_grad)
        if grads is not None:
            a.d_shape, a.d_expression, a.d_pose, a.d_neck_pose, a.d_transl, a.d_enlargement = map(p, grads)
        a.workspace, a.workspace_bytes = p(workspace), workspace.numel()
        return a

    def _launch(self, name: str, args) -> None:
        with torch.cuda.device(self.device):
            _lib.check(getattr(_lib.lib(), name)(C.byref(args), torch.cuda.current_stream(self.device).cuda_stream), name)

    def workspace(self) -> torch.Tensor:
        return torch.empty(self._ws_bytes, dtype=torch.uint8, device=self.device)

    def _check_params(self, shape, expression, pose, neck_pose, transl):
        for name, x, n in (("shape_params", shape, self.n_shape), ("expression_params", expression, self.n_exp),
                           ("pose_params", pose, 6), ("neck_pose", neck_pose, 3), ("transl", transl, 3)):
            if x.numel() != n or (x.dim() == 2 and x.shape[0] != 1):
                raise ValueError(f"NativeFlame: {name} must hold {n} values for one frame; got {tuple(x.shape)}")
            if x.device != self.device or x.dtype != torch.float32:
                raise ValueError(f"NativeFlame: {name} must be float32 on {self.device}")

    def __call__(self, shape_params=None, expression_params=None, pose_params=None, neck_pose=None, eye_pose=None, transl=None):
        """FLAME.forward (FLAME.py:204-248) without landmarks: (vertices [1,V,3], None).  neck_pose / transl default to zero
        as the module's own zero parameters; eye_pose stays at FLAME's zero default (a given one is refused)."""
        if eye_pose is not None:
            raise ValueError("NativeFlame: the eye pose is fixed at zero (FLAME's default); eye_pose is not supported")
        z = lambda n: torch.zeros(1, n, dtype=torch.float32, device=self.device)
        neck_pose = z(3) if neck_pose is None else neck_pose
        transl = z(3) if transl is None else transl
        self._check_params(shape_params, expression_params, pose_params, neck_pose, transl)
        return _LbsFunction.apply(self, shape_params, expression_params, pose_params, neck_pose, transl)[None], None

    def bind(self, model) -> "BoundFlame":
        """The forward into model.vertices (zeroing model.vertices.grad) and the backward from model.vertices.grad into the
        six FLAME tensors' .grad, with the argument blocks built once (FlameTrainer's sync-free path)."""
        return BoundFlame(self, model)


class BoundFlame:
    def __init__(self, flame: NativeFlame, model):
        names = ("_flame_shape", "_flame_exp", "_flame_pose", "_flame_neck_pose", "_flame_trans", "_vertices_enlargement")
        ps = [getattr(model, n) for n in names]
        flame._check_params(*ps[:5])
        if tuple(ps[5].shape) != (flame.V, 3) or tuple(model.vertices.shape) != (flame.V, 3):
            raise ValueError(f"NativeFlame.bind: the model's mesh must have the driver's {flame.V} vertices")
        for n, p in zip(names, ps):
            if p.grad is None or not p.is_contiguous() or not p.grad.is_contiguous():
                raise ValueError(f"NativeFlame.bind: {n} needs a contiguous tensor and gradient slot")
        self.flame, self.model = flame, model
        self.ws = flame.workspace()
        data = [p.detach() for p in ps]
        self.args = flame._args(*data, self.ws, vertices=model.vertices, vertices_grad=model.vertices.grad,
                                grads=[p.grad for p in ps])

    def forward(self) -> None:
        self.flame._launch("gms_flame_lbs_forward", self.args)

    def backward(self) -> None:
        self.flame._launch("gms_flame_lbs_backward", self.args)


class _LbsFunction(torch.autograd.Function):
    """FLAME's raw vertices o [V,3] (before transform_vertices_function): the kernels run with a unit enlargement, and their
    (o_x, -o_z, o_y) is permuted back, which is exact."""

    @staticmethod
    def forward(ctx, flame, shape, expression, pose, neck_pose, transl):
        flat = [x.detach().reshape(-1).contiguous() for x in (shape, expression, pose, neck_pose, transl)]
        ws = flame.workspace()
        out = torch.empty(flame.V, 3, dtype=torch.float32, device=flame.device)
        flame._launch("gms_flame_lbs_forward", flame._args(*flat, flame._ones, ws, vertices=out))
        ctx.flame, ctx.ws, ctx.shapes = flame, ws, [x.shape for x in (shape, expression, pose, neck_pose, transl)]
        ctx.save_for_backward(*flat)
        return torch.stack((out[:, 0], out[:, 2], -out[:, 1]), 1)

    @staticmethod
    def backward(ctx, g):
        flame = ctx.flame
        flat = ctx.saved_tensors
        gout = torch.stack((g[:, 0], -g[:, 2], g[:, 1]), 1).float().contiguous()
        grads = [torch.empty_like(x) for x in flat] + [torch.empty(flame.V, 3, dtype=torch.float32, device=flame.device)]
        flame._launch("gms_flame_lbs_backward", flame._args(*flat, flame._ones, ctx.ws, vertices_grad=gout, grads=grads))
        return (None,) + tuple(d.view(s) for d, s in zip(grads[:5], ctx.shapes))


# ---- FLAME's model pickle without its dependencies

class _Stand:
    """A pickled object of a class that is not imported (a chumpy array, a scipy sparse matrix): its state, kept as given."""
    kind = ""

    def __new__(cls, *args, **kwargs):
        return object.__new__(cls)

    def __init__(self, *args, **kwargs):
        pass

    def __setstate__(self, state):
        self.state = state


class _ModelUnpickler(pickle.Unpickler):
    def find_class(self, module, name):
        if module.startswith("scipy.sparse"):
            return type(name, (_Stand,), {"kind": "sparse", "fmt": name[:3]})
        if module.startswith("chumpy"):
            return type(name, (_Stand,), {"kind": "chumpy"})
        return super().find_class(module, name)


def _state_dict(obj) -> dict:
    st = getattr(obj, "state", None)
    if isinstance(st, tuple):        # (dict state, slot state)
        st = next((s for s in st if isinstance(s, dict)), None)
    return st if isinstance(st, dict) else {}


def _to_array(x, key: str) -> np.ndarray:
    """A model-file entry as a dense ndarray: arrays as they are, chumpy arrays from their pickled `x`, scipy sparse
    matrices rebuilt from data / indices / indptr and the shape.  Anything else fails, naming the key."""
    if isinstance(x, np.ndarray):
        return x
    if isinstance(x, _Stand):
        st = _state_dict(x)
        if x.kind == "chumpy":
            a = st.get("x")
            if isinstance(a, np.ndarray):
                return a
        elif x.kind == "sparse" and x.fmt in ("csc", "csr"):
            shape = st.get("_shape", st.get("shape"))
            data, indices, indptr = st.get("data"), st.get("indices"), st.get("indptr")
            if shape is not None and all(isinstance(a, np.ndarray) for a in (data, indices, indptr)):
                n_rows, n_cols = (int(s) for s in shape)
                dense = np.zeros((n_rows, n_cols), dtype=data.dtype)
                for k in range(len(indptr) - 1):
                    sl = slice(int(indptr[k]), int(indptr[k + 1]))
                    if x.fmt == "csc":
                        np.add.at(dense[:, k], indices[sl], data[sl])
                    else:
                        np.add.at(dense[k], indices[sl], data[sl])
                return dense
    raise ValueError(f"FLAME model file: no array could be found for {key!r} ({type(x).__name__})")
