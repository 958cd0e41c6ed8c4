"""Render and evaluate views natively: one gms_render_frame (gs_mesh) or gms_points_render_frame (gs_points pseudo-mesh)
call per view, no host synchronisation.

    renderer = NativeRenderer(model, W, H)
    image, radii, invdepth = renderer.render(cam, bg)                  # scripts/render.py, render_time_animated.py
    result = renderer.evaluate(test_cams, test_gts, bg)               # training_report / metrics.py

    renderer = PointsRenderer(PointsModel.from_flat_checkpoint(ply), W, H)
    image, radii, invdepth = renderer.render(cam, bg, triangles=transform_hotdog(renderer.model.triangles, t))
                                                                       # scripts/render_points_time_animated.py

    renderer = MeshBoundPointsRenderer(points_model.bind_to_mesh(*io_obj.read_obj(mesh_obj)), W, H)
    image, radii, invdepth = renderer.render(cam, bg, vertices=edited_vertices)
                                                                       # scripts/edit_pseudomesh_based_on_estimated_mesh.py

The first render learns N through one 4-byte read-back; every later one is sync-free, with the binning capacity predicted
per view (SyncFreeCapacity).  An overflowed render (N above its capacity) gives the background image and is counted in
`overflows`; the view's next render is sized from its true N.  evaluate() never reports an overflowed view's score: it
re-renders those views before it reads its results."""
from __future__ import annotations

import contextlib
from dataclasses import dataclass
from typing import List, Optional, Sequence

import torch

from . import _lib, io_image
from .capacity import SyncFreeCapacity, check_float32, grow_only_alloc
from .metrics import METRIC_NAMES, image_metrics, scratch_bytes


@dataclass
class Evaluation:
    per_view: torch.Tensor      # float64 [n,4] on the host, columns METRIC_NAMES
    mean: torch.Tensor          # float64 [4]: the mean of the per-view values (PSNR too, as both reference scripts average it)
    rerun: List[int]            # views whose first render overflowed its capacity and was re-rendered before scoring
    lpips: Optional[torch.Tensor] = None    # float32 [n] on the host: per-view LPIPS when evaluate() was given an Lpips


class NativeRenderer(SyncFreeCapacity):
    """Forward-only renders of one model at one image size.  The outputs of render() are buffers the renderer owns and the
    next call overwrites in stream order (ImageSink.write and anything else queued on the same stream read them first).
    A FlameGaussianModel is drawn at its `vertices`, which FlameTrainer.step leaves at the pose that step rendered (before
    its Adam update); call model.refresh_vertices() first to draw the current parameters (FlameTrainer.evaluate does)."""

    def __init__(self, model, width: int, height: int):
        self.model, self.W, self.H = model, int(width), int(height)
        dev, P = self._adopt(model)
        self.dev = dev
        self.ws = torch.empty(int(self._workspace_bytes(P)), dtype=torch.uint8, device=dev)
        self.image = torch.empty(3, self.H, self.W, dtype=torch.float32, device=dev)
        self.invdepth = torch.empty(1, self.H, self.W, dtype=torch.float32, device=dev)
        self.radii = torch.empty(P, dtype=torch.int32, device=dev)
        self._init_capacity(True)
        self._scratch, self._cb = grow_only_alloc(dev)
        self._metric_scratch = torch.empty(scratch_bytes(3, self.H, self.W), dtype=torch.uint8, device=dev)
        self._gt_u8 = io_image.GroundTruthBuffer(self.H, self.W, dev)

    def _adopt(self, model):
        """(device, Gaussian count) of the model this renderer draws; makes its face indices int64 and contiguous."""
        if model.faces.dtype != torch.int64 or not model.faces.is_contiguous():
            model.faces = model.faces.long().contiguous()
        return model.vertices.device, model._scale.shape[0]

    def _workspace_bytes(self, P: int) -> int:
        return _lib.lib().gms_render_workspace_bytes(P, self.W, self.H)

    @property
    def stale(self) -> bool:
        """The model no longer has the Gaussian count this renderer was sized for (densification changed it): a new
        renderer has to draw it."""
        return self._adopt(self.model)[1] != self.radii.shape[0]

    def _features(self) -> torch.Tensor:
        m = self.model
        f = m._features if m._features is not None else m.get_features      # packed SH: zero-copy
        return f.detach().contiguous()

    _sweep_vertices = None      # set by render(vertices=...) for that one frame

    def _check(self, cam, bg) -> None:
        m = self.model
        for name in ("vertices", "_alpha", "_scale", "_opacity"):
            check_float32(getattr(m, name), f"NativeRenderer: model.{name}", self.dev)
        v = self._sweep_vertices
        if v is not None:
            check_float32(v, "NativeRenderer: the frame's vertices", self.dev)
            if v.shape != m.vertices.shape:
                raise RuntimeError(f"NativeRenderer: the frame's vertices must be {list(m.vertices.shape)}; got {list(v.shape)}")
        if m.faces.device != self.dev:
            raise RuntimeError("NativeRenderer: model.faces must live on the model's device")
        if m._scale.shape[0] != self.radii.shape[0]:
            raise RuntimeError("NativeRenderer: the model's Gaussian count changed; make a new renderer")
        self._check_view(cam, bg)

    def _render(self, cam, bg, scale_modifier: float, antialiasing: bool, capacity: int = None, n_host: int = None) -> None:
        """One gms_render_frame into the renderer's buffers: sync-free at `capacity` with (N, flag) at the mapped address
        `n_host` when given, else as SyncFreeCapacity._launch decides."""
        self._check(cam, bg)
        m = self.model
        feats = self._features()
        a = _lib.RenderArgs()
        v = m.vertices if self._sweep_vertices is None else self._sweep_vertices
        a.V, a.M = v.shape[0], feats.shape[1]
        a.F, a.K, seg = m.frame_sizes()
        if seg is not None:
            a.segments, a.n_segments = seg, len(seg)
        a.vertices, a.faces, a.alpha_raw, a.scale_raw = v.data_ptr(), m.faces.data_ptr(), m._alpha.data_ptr(), m._scale.data_ptr()
        a.features, a.opacity_raw, a.eps = feats.data_ptr(), m._opacity.data_ptr(), m.eps_s0
        a.alpha_activation = getattr(m, "alpha_activation", _lib.ALPHA_RELU)
        self._call("gms_render_frame", a, cam, bg, scale_modifier, antialiasing, capacity, n_host)

    def _call(self, fn: str, a, cam, bg, scale_modifier: float, antialiasing: bool, capacity: int, n_host: int) -> None:
        """Points `a`'s outputs at the renderer's buffers and issues `fn`."""
        a.image, a.invdepth, a.radii = self.image.data_ptr(), self.invdepth.data_ptr(), self.radii.data_ptr()
        self._launch(fn, a, cam, bg, scale_modifier, antialiasing, capacity, n_host, debug=self._debug)

    _debug = False      # set by render(debug=...) / evaluate(debug=...) for that call

    @contextlib.contextmanager
    def _debug_mode(self, debug: bool):
        self._debug = bool(debug)
        try:
            yield
        finally:
            self._debug = False

    def render(self, cam, bg: torch.Tensor, scale_modifier: float = 1.0, antialiasing: bool = False,
               vertices: torch.Tensor = None, debug: bool = False):
        """(image [3,H,W], radii [P], invdepth [1,H,W]) of one view, the reference's render(...)["render"], ["radii"],
        ["depth"].  `vertices` (float32, model.vertices' shape), when given, is this frame's mesh in place of the model's
        (one frame of an animated sweep, renderer/gaussian_animated_renderer's `triangles` as vertices[faces]); the model
        is never modified.  debug: the reference's pipe.debug (every launch of the frame waited for and named on a fault,
        the binning check on the frame's buffers)."""
        self._sweep_vertices = None if vertices is None else vertices.detach()
        try:
            with self._debug_mode(debug):
                self._render(cam, bg, scale_modifier, antialiasing)
        finally:
            self._sweep_vertices = None
        return self.image, self.radii, self.invdepth

    def _gt_float(self, gt: torch.Tensor) -> torch.Tensor:
        """float [3,H,W] as is; uint8 [H,W,3] (8-bit ground truth) -> byte / 255 in one reused device buffer."""
        if gt.dtype == torch.uint8:
            return self._gt_u8(gt, "evaluate")
        if tuple(gt.shape) != (3, self.H, self.W) or gt.dtype != torch.float32:
            raise ValueError(f"evaluate: float ground truth must be float32 [3,{self.H},{self.W}]; got {gt.dtype} {tuple(gt.shape)}")
        return gt.to(self.dev, non_blocking=True)

    def evaluate(self, cams: Sequence, gts: Sequence[torch.Tensor], bg: torch.Tensor, protocol: str = "training_report",
                 scale_modifier: float = 1.0, antialiasing: bool = False, lpips=None, debug: bool = False) -> Evaluation:
        """Renders every view and scores it against its ground truth (metrics.METRIC_NAMES under `protocol`, "training_report"
        or "metrics"), all on the current stream into one device array; the host synchronises once, at the end.  Views whose
        render overflowed its predicted capacity are then re-rendered, sized from their true N, and re-scored before the
        array is read.  Given an lpips.Lpips (protocol "metrics" only, as metrics.py alone reports LPIPS), each view's LPIPS
        is scored in the same pass on the 8-bit round trip of the render and of the ground truth, into Evaluation.lpips.
        debug: every view renders in the reference's debug mode (render)."""
        with self._debug_mode(debug):
            return self._evaluate(cams, gts, bg, protocol, scale_modifier, antialiasing, lpips)

    def _evaluate(self, cams, gts, bg, protocol, scale_modifier, antialiasing, lpips) -> Evaluation:
        if len(cams) != len(gts):
            raise ValueError(f"evaluate: {len(cams)} cameras but {len(gts)} ground-truth images")
        if lpips is not None and protocol != "metrics":
            raise ValueError(f"evaluate: LPIPS is scored under protocol 'metrics' only (metrics.py); got {protocol!r}")
        n = len(cams)
        out = torch.empty(n, len(METRIC_NAMES), dtype=torch.float64, device=self.dev)
        lp = torch.empty(n, 6, dtype=torch.float32, device=self.dev) if lpips is not None else None
        slots = torch.full((max(n, 1), 2), -1, dtype=torch.int32).pin_memory()     # per view: (N, overflow flag), mapped
        slots_np = slots.numpy()
        keys = [self._view_key(c) for c in cams]
        caps = []

        def one(v, capacity):
            self._render(cams[v], bg, scale_modifier, antialiasing, capacity, slots.data_ptr() + 8 * v)
            gt = self._gt_float(gts[v])
            image_metrics(self.image, gt, protocol, out=out[v], scratch=self._metric_scratch)
            if lp is not None:
                lpips.lpips(self._round_trip(self.image, 0), self._round_trip(gt, 1), out=lp[v])

        for v in range(n):
            caps.append(self._predict_capacity(keys[v]))
            one(v, caps[v])
        torch.cuda.current_stream(self.dev).synchronize()
        rerun = []
        for v in range(n):
            nv = int(slots_np[v, 0])
            self._note(keys[v], nv)
            if nv > caps[v]:
                self.overflows += 1
                rerun.append(v)
        for v in rerun:
            one(v, max(int(slots_np[v, 0]), 1))
        if n:
            self.capacity = max(caps)
        lp_host = None
        if lp is not None:          # ordered before the read-back below, which waits for it
            lp_host = torch.empty(n, dtype=torch.float32).pin_memory()
            lp_host.copy_(lp[:, 5], non_blocking=True)
        per_view = out.cpu()        # (waits for the re-runs, if any)
        mean = per_view.mean(0) if n else torch.full((len(METRIC_NAMES),), float("nan"), dtype=torch.float64)
        return Evaluation(per_view=per_view, mean=mean, rerun=rerun, lpips=lp_host)

    def _round_trip(self, image: torch.Tensor, slot: int) -> torch.Tensor:
        """save_image's 8-bit rounding of float [3,H,W] and back to byte / 255 (what metrics.py reads from the PNG), into one
        of two reused device buffers."""
        if getattr(self, "_rt", None) is None:
            self._rt = (torch.empty(self.H, 3 * self.W, dtype=torch.uint8, device=self.dev),
                        [torch.empty(3, self.H, self.W, dtype=torch.float32, device=self.dev) for _ in range(2)])
        u8, f = self._rt
        io_image.quantize(image, out=u8)
        return io_image.to_device_float(u8.view(self.H, self.W, 3), out=f[slot])


class PointsRenderer(NativeRenderer):
    """NativeRenderer for a gs_points pseudo-mesh model (model.PointsModel): every render derives the Gaussians from the
    triangles inside gms_points_render_frame.  evaluate(), the capacity prediction and the overflow re-runs are
    NativeRenderer's."""

    _frame_triangles = None     # set by render(triangles=...) for that one frame

    def _adopt(self, model):
        return model.triangles.device, model.triangles.shape[0]

    def _workspace_bytes(self, P: int) -> int:
        return _lib.lib().gms_points_render_workspace_bytes(P, self.W, self.H)

    def _check(self, cam, bg) -> None:
        m = self.model
        for name, t in (("triangles", self._triangles), ("_features", m._features), ("_opacity", m._opacity)):
            check_float32(t, f"PointsRenderer: {name}", self.dev)
        P = self.radii.shape[0]
        if tuple(self._triangles.shape) != (P, 3, 3) or m._features.shape[0] != P or tuple(m._opacity.shape) != (P, 1):
            raise RuntimeError(f"PointsRenderer: sized for {P} Gaussians: triangles must be [{P},3,3], features [{P},M,3], "
                               f"opacity [{P},1]; got {tuple(self._triangles.shape)}")
        self._check_view(cam, bg)

    def _render(self, cam, bg, scale_modifier: float, antialiasing: bool, capacity: int = None, n_host: int = None) -> None:
        m = self.model
        self._check(cam, bg)
        a = _lib.PointsRenderArgs()
        a.P, a.M = self.radii.shape[0], m._features.shape[1]
        a.triangles, a.features, a.opacity_raw, a.eps = self._triangles.data_ptr(), m._features.data_ptr(), m._opacity.data_ptr(), m.eps_s0
        self._call("gms_points_render_frame", a, cam, bg, scale_modifier, antialiasing, capacity, n_host)

    @property
    def _triangles(self) -> torch.Tensor:
        return self.model.triangles if self._frame_triangles is None else self._frame_triangles

    def render(self, cam, bg: torch.Tensor, triangles: torch.Tensor = None, scale_modifier: float = 1.0, antialiasing: bool = False,
               debug: bool = False):
        """(image [3,H,W], radii [P], invdepth [1,H,W]) of one view.  `triangles` [P,3,3], when given, are this frame's
        pseudo-mesh in place of the model's (the `triangles` argument of renderer/gaussian_points_animated_renderer's
        render); the model is never modified.  (The reference's render calls pc.prepare_scaling_rot(triangles), which
        overwrites pc._scaling and pc._rotation with those of the frame's triangles.)"""
        self._frame_triangles = None if triangles is None else triangles.detach()
        try:
            return super().render(cam, bg, scale_modifier=scale_modifier, antialiasing=antialiasing, debug=debug)
        finally:
            self._frame_triangles = None


class MeshBoundPointsRenderer(NativeRenderer):
    """NativeRenderer for a pseudo-mesh bound to a driving mesh (model.MeshBoundPointsModel): every render re-poses the
    pseudo-triangles from a pose of that mesh and derives the Gaussians from them inside ONE kernel of
    gms_bound_points_render_frame; the triangles are never written.  Gaussians whose face is degenerate in the pose are not
    drawn (radius 0).  evaluate(), the capacity prediction and the overflow re-runs are NativeRenderer's."""

    _frame_vertices = None      # set by render(vertices=...) for that one frame

    def _adopt(self, model):
        return model.binding.face.device, model.binding.P

    def _workspace_bytes(self, P: int) -> int:
        return _lib.lib().gms_bound_points_render_workspace_bytes(P, self.W, self.H)

    def _check(self, cam, bg) -> None:
        m, b = self.model, self.model.binding
        P = self.radii.shape[0]
        for name, t in (("_features", m._features), ("_opacity", m._opacity), ("binding.coeffs", b.coeffs)):
            check_float32(t, f"MeshBoundPointsRenderer: {name}", self.dev)
        if b.P != P or m._features.shape[0] != P or tuple(m._opacity.shape) != (P, 1):
            raise RuntimeError(f"MeshBoundPointsRenderer: sized for {P} Gaussians: features must be [{P},M,3], opacity [{P},1]")
        v = m.vertices if self._frame_vertices is None else self._frame_vertices
        if not (torch.is_tensor(v) and v.is_cuda and v.dtype == torch.float32 and v.is_contiguous() and v.device == self.dev
                and tuple(v.shape) == (b.V, 3)):
            raise RuntimeError(f"MeshBoundPointsRenderer: the pose `vertices` must be a contiguous float32 [{b.V},3] CUDA "
                               f"tensor on {self.dev}")
        for name, t in (("binding.face", b.face), ("binding.faces", b.faces)):
            if not (t.is_cuda and t.is_contiguous() and t.device == self.dev):
                raise RuntimeError(f"MeshBoundPointsRenderer: {name} must be a contiguous CUDA tensor on {self.dev}")
        self._check_view(cam, bg)

    def _render(self, cam, bg, scale_modifier: float, antialiasing: bool, capacity: int = None, n_host: int = None) -> None:
        m, b = self.model, self.model.binding
        self._check(cam, bg)
        v = m.vertices if self._frame_vertices is None else self._frame_vertices
        a = _lib.BoundPointsRenderArgs()
        a.P, a.M = self.radii.shape[0], m._features.shape[1]
        a.face, a.coeffs, a.V, a.F = b.face.data_ptr(), b.coeffs.data_ptr(), b.V, b.faces.shape[0]
        a.vertices, a.faces = v.data_ptr(), b.faces.data_ptr()
        a.features, a.opacity_raw, a.eps = m._features.data_ptr(), m._opacity.data_ptr(), m.eps_s0
        self._call("gms_bound_points_render_frame", a, cam, bg, scale_modifier, antialiasing, capacity, n_host)

    def render(self, cam, bg: torch.Tensor, vertices: torch.Tensor = None, scale_modifier: float = 1.0, antialiasing: bool = False,
               debug: bool = False):
        """(image [3,H,W], radii [P], invdepth [1,H,W]) of one view.  `vertices` [V,3], when given, is this frame's pose of
        the driving mesh in place of the model's (an edited mesh, or one frame of an animation); the model is never
        modified."""
        self._frame_vertices = None if vertices is None else self.model.binding.check_vertices(vertices)
        try:
            return super().render(cam, bg, scale_modifier=scale_modifier, antialiasing=antialiasing, debug=debug)
        finally:
            self._frame_vertices = None


class RendererSet:
    """The renderers of one model's views at any image sizes: one cls(model, W, H) per size, made when a view of that size
    first needs one, all sized for the Gaussian count P they were made at (a trainer makes a new set when P changes)."""

    def __init__(self, cls, model, P: int):
        self.cls, self.model, self.P = cls, model, int(P)
        self.by_size = {}

    def for_view(self, cam):
        """The renderer of `cam`'s image size."""
        size = (int(cam.image_width), int(cam.image_height))
        if size not in self.by_size:
            self.by_size[size] = self.cls(self.model, *size)
        return self.by_size[size]

    def render(self, cam, bg: torch.Tensor, **kw):
        """for_view(cam).render(cam, bg, **kw)."""
        return self.for_view(cam).render(cam, bg, **kw)

    def evaluate(self, cams: Sequence, gts: Sequence[torch.Tensor], bg: torch.Tensor, **kw) -> Evaluation:
        """NativeRenderer.evaluate over views of any sizes: each size's views through that size's renderer (one host
        synchronisation per size).  per_view, rerun and lpips are in view order; the mean is per_view's, in float64 on the
        host."""
        if len(cams) != len(gts):
            raise ValueError(f"evaluate: {len(cams)} cameras but {len(gts)} ground-truth images")
        groups = {}
        for v, cam in enumerate(cams):
            groups.setdefault((int(cam.image_width), int(cam.image_height)), []).append(v)
        if len(groups) <= 1:
            return self.for_view(cams[0]).evaluate(cams, gts, bg, **kw)
        per_view = torch.empty(len(cams), len(METRIC_NAMES), dtype=torch.float64)
        rerun, lpips = [], None
        for views in groups.values():
            e = self.for_view(cams[views[0]]).evaluate([cams[v] for v in views], [gts[v] for v in views], bg, **kw)
            per_view[views] = e.per_view
            rerun += [views[i] for i in e.rerun]
            if e.lpips is not None:
                lpips = torch.empty(len(cams), dtype=torch.float32) if lpips is None else lpips
                lpips[views] = e.lpips
        return Evaluation(per_view=per_view, mean=per_view.mean(0), rerun=sorted(rerun), lpips=lpips)


def render_points_frame(model, cam, bg: torch.Tensor, triangles: torch.Tensor = None, scale_modifier: float = 1.0,
                        antialiasing: bool = False):
    """The same render through the autograd shim, as renderer/gaussian_points_animated_renderer/__init__.py:21-114 does it
    on the library's kernels: expansion.points_prepare_scaling_rot(activated=True), an ATen sigmoid and GaussianRasterizer
    (whose forward reads N back to the host).  Returns (image, radii, invdepth)."""
    import diff_gaussian_rasterization as dgr
    from . import expansion
    tri = model.triangles if triangles is None else triangles
    xyz, scales, rots = expansion.points_prepare_scaling_rot(tri, model.eps_s0, activated=True)
    rs = dgr.GaussianRasterizationSettings(
        image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
        bg=bg, scale_modifier=float(scale_modifier), viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
        sh_degree=model.active_sh_degree, campos=cam.camera_center, prefiltered=False, debug=False, antialiasing=antialiasing)
    return dgr.GaussianRasterizer(raster_settings=rs)(means3D=xyz, means2D=torch.zeros_like(xyz), opacities=model.get_opacity,
                                                      shs=model.get_features, scales=scales, rotations=rots)


class NativeFreeRenderer(NativeRenderer):
    """NativeRenderer for free Gaussians (model.FreeGaussianModel, gs / gs_flat): every render activates the raw parameters
    inside gms_free_render_frame.  evaluate(), the capacity prediction and the overflow re-runs are NativeRenderer's."""

    def _adopt(self, model):
        return model._xyz.device, model.P

    def _check(self, cam, bg) -> None:
        m = self.model
        for name in m.NAMES:
            check_float32(getattr(m, name), f"NativeFreeRenderer: model.{name}", self.dev)
        if m.P != self.radii.shape[0]:
            raise RuntimeError("NativeFreeRenderer: the model's Gaussian count changed; make a new renderer")
        self._check_view(cam, bg)

    def _render(self, cam, bg, scale_modifier: float, antialiasing: bool, capacity: int = None, n_host: int = None) -> None:
        m = self.model
        self._check(cam, bg)
        a = _lib.FreeRenderArgs()
        a.P, a.M, a.scale_cols = m.P, m._features.shape[1], m.scale_cols
        a.xyz, a.scaling_raw, a.rotation_raw = m._xyz.data_ptr(), m._scaling.data_ptr(), m._rotation.data_ptr()
        a.features, a.opacity_raw, a.eps = m._features.data_ptr(), m._opacity.data_ptr(), m.eps_s0
        self._call("gms_free_render_frame", a, cam, bg, scale_modifier, antialiasing, capacity, n_host)


class FlameRenderer(NativeRenderer):
    """Renders of a trained gs_flame checkpoint (model.FlameCheckpoint) by the protocol of scripts/render_flame.py, in ONE call
    per view (gms_flame_render_frame): xyz from the stored activated weights and a driving pose, scales and rotations from
    the checkpoint's rows (they do not follow the pose, as in the reference).  evaluate(), the capacity prediction and the
    overflow re-runs are NativeRenderer's; evaluate() draws the checkpoint's `vertices` pose."""

    _frame_vertices = None

    def _adopt(self, model):
        return model.alpha.device, model.P

    def _workspace_bytes(self, P: int) -> int:
        return _lib.lib().gms_flame_render_workspace_bytes(P, self.W, self.H)

    def _check(self, cam, bg) -> None:
        m = self.model
        v = m.vertices if self._frame_vertices is None else self._frame_vertices
        V = m._vertices_enlargement.shape[0]
        if not (torch.is_tensor(v) and v.is_cuda and v.dtype == torch.float32 and v.is_contiguous() and v.device == self.dev
                and tuple(v.shape) == (V, 3)):
            raise RuntimeError(f"FlameRenderer: the pose `vertices` must be a contiguous float32 [{V},3] CUDA tensor on {self.dev}")
        for name in ("alpha", "_scaling", "_rotation", "_features", "_opacity"):
            check_float32(getattr(m, name), f"FlameRenderer: {name}", self.dev)
        if m.P != self.radii.shape[0]:
            raise RuntimeError("FlameRenderer: the checkpoint's Gaussian count changed; make a new renderer")
        self._check_view(cam, bg)

    def _render(self, cam, bg, scale_modifier: float, antialiasing: bool, capacity: int = None, n_host: int = None) -> None:
        m = self.model
        self._check(cam, bg)
        v = m.vertices if self._frame_vertices is None else self._frame_vertices
        a = _lib.FlameRenderArgs()
        a.V, a.F, a.K, a.M = v.shape[0], m.alpha.shape[0], m.alpha.shape[1], m._features.shape[1]
        a.vertices, a.faces, a.alpha = v.data_ptr(), m.faces.data_ptr(), m.alpha.data_ptr()
        a.scaling_log, a.rotation_raw = m._scaling.data_ptr(), m._rotation.data_ptr()
        a.features, a.opacity_raw = m._features.data_ptr(), m._opacity.data_ptr()
        self._call("gms_flame_render_frame", a, cam, bg, scale_modifier, antialiasing, capacity, n_host)

    def render(self, cam, bg: torch.Tensor, vertices: torch.Tensor = None, scale_modifier: float = 1.0, antialiasing: bool = False,
               debug: bool = False):
        """(image [3,H,W], radii [P], invdepth [1,H,W]) of one view at the pose `vertices` [V,3] (default: the checkpoint's
        `vertices`); the checkpoint is never modified."""
        self._frame_vertices = None if vertices is None else vertices.detach().float().contiguous()
        try:
            return super().render(cam, bg, scale_modifier=scale_modifier, antialiasing=antialiasing, debug=debug)
        finally:
            self._frame_vertices = None
