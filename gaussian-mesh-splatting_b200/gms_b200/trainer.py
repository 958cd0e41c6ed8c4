"""One optimisation step of gs_mesh on the H100-native path, single GPU or frame-sharded data parallel.

Step structure = train.py:89-157 of the reference: pick a camera, render (expansion + rasterizer), loss
(train.py:105-107), backward (train.py:108), optimizer step (train.py:146-148), re-expand (train.py:154-157 -- here the
expansion is simply the first thing the next step's render does, in one fused launch).

Multi-GPU (the reference has none, SURVEY.md 2.1): one process per GPU, every rank holds a replica of the mesh-Gaussian
parameters, rank r renders camera `step*world + r` of the schedule, and ONE NCCL all-reduce per step averages the
flattened gradient of the shared parameters (vertices, _alpha, _scale, _features_dc, _features_rest, _opacity).
All gradients live in ONE contiguous buffer (param.grad are views into it), so the collective is a single call.
"""
from __future__ import annotations

import contextlib
import math
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

import diff_gaussian_rasterization as dgr

from . import _lib, debug as _debug
from .anomaly import FRAME_STAGES, AnomalyError, AnomalyRecord, layout_of
from .capacity import SyncFreeCapacity, check_float32, grow_only_alloc, recorded_event
from .flame import NativeFlame
from .io_image import GroundTruthBuffer
from .losses import fused_training_loss
from .model import MeshGaussianModel
from .optim import FlatAdam, mesh_model_groups
from .render import NativeFreeRenderer, NativeRenderer, RendererSet
from .scenes import Camera


def shard_cameras(n_cameras: int, step: int, rank: int, world: int) -> int:
    """Camera index rank `rank` renders at `step`: consecutive cameras of the schedule go to consecutive ranks."""
    return (step * world + rank) % n_cameras


def render_frame(model: MeshGaussianModel, cam: Camera, bg: torch.Tensor, fused: bool = True, antialiasing: bool = False):
    """Expansion + rasterizer forward for one camera.  Returns (image, radii, invdepth)."""
    if fused:
        xyz, scales, rots = model.expand_fused(activated=True)
    else:   # the reference's two-step protocol + getters
        model.update_alpha(); model.prepare_scaling_rot()
        xyz, scales, rots = model.get_xyz, model.get_scaling, model.get_rotation
    rs = dgr.GaussianRasterizationSettings(
        image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
        bg=bg, scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
        sh_degree=model.active_sh_degree, campos=cam.camera_center, prefiltered=False, debug=False, antialiasing=antialiasing)
    means2D = torch.zeros_like(xyz, requires_grad=xyz.requires_grad)
    return dgr.GaussianRasterizer(raster_settings=rs)(means3D=xyz, means2D=means2D, opacities=model.get_opacity,
                                                      shs=model.get_features, scales=scales, rotations=rots)


class _FrameSize(SyncFreeCapacity):
    """The image sizes a training frame runs.  An exact-size frame (up_to=False) runs W x H views only.  An up_to frame
    runs every view of at most W x H at the view's own size, in ONE workspace of gms_frame_workspace_bytes(P, W, H):
    gms_train_frame and gms_free_train_frame lay out the image-sized part of the workspace, the loss scratch and the
    rasterizer's per-pixel scratch from the size in each call's settings, and each of those layouts for w x h <= W x H
    fits in the one for W x H (their byte counts grow with w and with h).  The ground truth of a smaller view fills the
    head of one W x H buffer.  The capacity prediction is per view, so views of different sizes keep their own N."""

    def _init_size(self, width: int, height: int, up_to: bool) -> None:
        self.W, self.H, self.up_to = int(width), int(height), bool(up_to)
        self._gt_u8 = GroundTruthBuffer(self.H, self.W, self.dev, up_to=self.up_to)

    def _fit_workspace(self) -> None:
        """A workspace for the model's current Gaussian count at W x H (kept when it is large enough)."""
        from . import _lib
        need = int(_lib.lib().gms_frame_workspace_bytes(self._gaussians(), self.W, self.H))
        if self.ws is None or self.ws.numel() < need:
            self.ws = None
            self.ws = torch.empty(need, dtype=torch.uint8, device=self.dev)

    def grow(self, width: int, height: int) -> None:
        """Run views of up to max(W, width) x max(H, height) from now on (an up_to frame).  When that is larger, the
        workspace and the ground-truth buffer grow and every view's next frame learns its N with one read-back."""
        W, H = max(self.W, int(width)), max(self.H, int(height))
        larger = (W, H) != (self.W, self.H)
        self._init_size(W, H, True)
        if larger:
            self._fit_workspace()
            self._forget_views()


class NativeFrame(_FrameSize):
    """One training frame through gms_train_frame: expansion, rasterizer, loss and both backward passes issued from ONE C
    call on the current stream -- no autograd graph, no per-op Python.  Gradients land in the parameters' preallocated
    .grad views (FlatAdam's flat buffer); intermediates live in a persistent workspace, rasterizer scratch in grow-only
    buffers served through the allocation callback.

    sync_free (default): only the FIRST frame learns N through the stock-style 4-byte read-back; from then on the binning
    region is sized per view by the capacity prediction of SyncFreeCapacity (gms_b200/capacity.py), and a frame whose N
    exceeds its capacity renders the background with zero gradients and is counted in `overflows`.

    up_to: width x height is the largest view; smaller views run at their own size in the same workspace (_FrameSize)."""

    def __init__(self, model: MeshGaussianModel, width: int, height: int, lambda_dssim: float = 0.2, sync_free: bool = True,
                 world: int = 1, rank: int = 0, up_to: bool = False):
        assert model._features is not None, "NativeFrame needs packed SH features"
        self.model, self.lam = model, float(lambda_dssim)
        dev = model.vertices.device
        self.dev = dev
        P = model._scale.shape[0]
        self._init_size(width, height, up_to)
        self.ws = None
        self._fit_workspace()
        self.view_size = (self.W, self.H)       # W x H of the last frame
        self.loss = torch.zeros(3, dtype=torch.float32, device=dev)
        self._init_capacity(sync_free)
        # factored SH gradient (run(..., factored=True)): slot r of `exchange` = [3P colour gradients | camera centre | pad] of
        # rank r's frame; this rank's frame writes slot `rank`, FlatAdam(sh_factored=True) all-gathers and consumes the rest
        self.world, self.rank = int(world), int(rank)
        self.slot = (3 * P + 3 + 63) // 64 * 64
        self.exchange = None
        self.ev_loss = None         # recorded by gms_train_frame right after the loss kernels (read_loss_async)
        self._loss_read, self._side = None, None
        self.ev_sh = None           # recorded by gms_train_frame right after the preprocess backward (world > 1: the exchange of the
                                    # colour gradients starts there, on the optimizer's communication stream)
        self._check_model()
        self._scratch, self._cb = grow_only_alloc(dev)

    def _gaussians(self) -> int:
        return self.model._scale.shape[0]

    def _check_model(self):
        """Raw pointers go straight to CUDA kernels: dtype / device / layout are checked here, once, instead of failing
        as an illegal address later."""
        m = self.model
        if m.faces.dtype != torch.int64 or not m.faces.is_contiguous():
            m.faces = m.faces.long().contiguous()
        for name in ("vertices", "_alpha", "_scale", "_features", "_opacity"):
            t = getattr(m, name)
            check_float32(t, f"NativeFrame: model.{name}", self.dev)
            if t.grad is None or not t.grad.is_contiguous() or t.grad.device != self.dev:
                raise RuntimeError(f"NativeFrame: model.{name}.grad must be a preallocated contiguous buffer (FlatAdam provides it)")
        if m.faces.device != self.dev:
            raise RuntimeError("NativeFrame: model.faces must live on the model's device")

    def read_loss_async(self, loss_host: torch.Tensor, loss_ready: Optional[torch.cuda.Event] = None) -> None:
        """Copy the last frame's loss into pinned host memory from a side stream as soon as the LOSS kernels are done (the
        event gms_train_frame records ~40 % into the frame), not after the whole frame: a caller that waits for `loss_ready`
        gets the value while the backward pass is still running and has that time to queue its next step.  The leading
        loss_host.numel() values of the frame's [loss, L1, SSIM] vector are copied (1: the loss; 2: the loss and L1)."""
        if self._side is None:
            self._side = torch.cuda.Stream(self.dev)
        self._side.wait_event(self.ev_loss)
        with torch.cuda.stream(self._side):
            loss_host.copy_(self.loss[:loss_host.numel()].reshape(loss_host.shape), non_blocking=True)
            if loss_ready is not None:
                loss_ready.record(self._side)
            self._loss_read = torch.cuda.Event()
            self._loss_read.record(self._side)

    def sh_factors(self) -> dict:
        """What FlatAdam.step(sh=...) needs after a factored frame."""
        import ctypes as C
        from . import _lib
        v = _lib.FrameView()
        _lib.check(_lib.lib().gms_frame_views(self.ws.data_ptr(), self.model._scale.shape[0], *self.view_size, C.byref(v)), "gms_frame_views")
        return dict(xyz=v.xyz, exchange=self.exchange, degree=self.model.active_sh_degree, event=self.ev_sh)

    def run(self, cam: Camera, gt: torch.Tensor, bg: torch.Tensor, factored: bool = False, sh_adam=None,
            antialiasing: bool = False, anomaly: Optional[AnomalyRecord] = None, anomaly_stages: int = FRAME_STAGES,
            debug: bool = False) -> torch.Tensor:
        """sh_adam (FlatAdam.begin_fused_sh_step()): the frame also applies the SH parameters' Adam step, and writes no SH
        gradient (unless `factored` asks for the colour gradient as well).  gt: float32 [3,H,W], or uint8 [H,W,3] (dequantized
        on the device into the frame's buffer).  antialiasing: the reference's pipe.antialiasing (each splat's opacity scaled
        by the ratio of its 2D covariance determinants before and after the low-pass dilation, forward and backward).
        anomaly: the frame scans the outputs of each backward stage selected in anomaly_stages (bits 1 << _lib.ANOMALY_*) for
        NaN into this record (not with sh_adam); the caller resets and reads it.  debug: the reference's pipe.debug (every
        launch waited for and named on a fault, the binning check on the frame's buffers, a violation raises)."""
        import ctypes as C
        from . import _lib
        if gt.dtype == torch.uint8:
            gt = self._gt_u8(gt, "NativeFrame.run")
            if debug:
                _debug.sync("gms_image_dequantize", self.dev)
        self._check_view(cam, bg, "NativeFrame.run", gt=gt, gt_fits=lambda W, H: tuple(gt.shape[-2:]) == (H, W))
        self.view_size = (int(cam.image_width), int(cam.image_height))
        if not gt.is_contiguous() or gt.dtype != torch.float32:
            gt = gt.contiguous().float()
        m = self.model
        a = _lib.FrameArgs()
        a.V, a.M = m.vertices.shape[0], m._features.shape[1]
        a.F, a.K, seg = m.frame_sizes()
        if seg is not None:
            a.segments, a.n_segments = seg, len(seg)
        a.vertices, a.faces, a.alpha_raw, a.scale_raw = m.vertices.data_ptr(), m.faces.data_ptr(), m._alpha.data_ptr(), m._scale.data_ptr()
        a.features, a.opacity_raw, a.eps = m._features.data_ptr(), m._opacity.data_ptr(), m.eps_s0
        a.alpha_activation = getattr(m, "alpha_activation", _lib.ALPHA_RELU)
        a.d_vertices, a.d_alpha_raw, a.d_scale_raw = m.vertices.grad.data_ptr(), m._alpha.grad.data_ptr(), m._scale.grad.data_ptr()
        a.d_features, a.d_opacity_raw = m._features.grad.data_ptr(), m._opacity.grad.data_ptr()
        if factored:        # no SH gradient rows: the colour gradient + camera centre go to this rank's exchange slot
            if self.exchange is None:
                self.exchange = torch.zeros(self.world, self.slot, dtype=torch.float32, device=self.dev)
            a.d_features, a.d_color_sh = None, self.exchange[self.rank].data_ptr()
            if self.world > 1:
                self.ev_sh = recorded_event(self.ev_sh, self.dev)
                a.event_sh_ready = self.ev_sh.cuda_event
        if sh_adam is not None:
            a.d_features = None
            a.sh_adam = C.pointer(sh_adam)
        self.ev_loss = recorded_event(self.ev_loss, self.dev)
        a.event_loss_ready = self.ev_loss.cuda_event
        if self._loss_read is not None:         # an asynchronous read-back of the previous frame's loss (read_loss_async) must be
            torch.cuda.current_stream(self.dev).wait_event(self._loss_read)     # done before this frame's loss kernels overwrite it
            self._loss_read = None
        a.gt, a.lambda_dssim, a.loss = gt.data_ptr(), self.lam, self.loss.data_ptr()
        if anomaly is not None:
            a.anomaly, a.anomaly_stages = anomaly.ptr, int(anomaly_stages)
        self._launch("gms_train_frame", a, cam, bg, antialiasing=antialiasing, **({"debug": True} if debug else {}))
        return self.loss[0]


def check_antialiasing(state: dict, antialiasing: bool, who: str) -> None:
    """Refuse a trainer state written with the other antialiasing setting, so a resumed run renders as it was trained.  A
    state without the entry was written before the setting was recorded, when every trainer ran without antialiasing."""
    saved = bool(state.get("antialiasing", False))
    if saved != antialiasing:
        raise ValueError(f"{who}.load_state_dict: the state was trained with antialiasing={saved}, but this trainer runs "
                         f"antialiasing={antialiasing}")


def anomaly_record(record: Optional[AnomalyRecord], dev) -> AnomalyRecord:
    """A trainer's anomaly record (`record`, or a new one on `dev`), reset for the next frame."""
    return (record or AnomalyRecord(dev)).reset()


def check_anomaly(record: AnomalyRecord, model, cam: Camera, opt, iteration: Optional[int] = None, restore=None) -> None:
    """Reads the step's anomaly record (one host synchronisation).  On a NaN, the step is undone before AnomalyError is
    raised: `restore()` (when given) puts back what the frame accumulated into, and the gradient buffer is zeroed (the vertex
    gradient accumulates across frames), so the trainer can take its next step."""
    try:
        record.check(layout_of(model, cam), iteration)
    except AnomalyError:
        if restore is not None:
            restore()
        opt.zero_grad()
        raise


def refuse_data_parallel_anomaly(detect_anomaly: bool, world: int, who: str) -> None:
    if detect_anomaly and world > 1:
        raise ValueError(f"{who}: detect_anomaly needs one GPU (world {world}): data-parallel anomaly detection is not implemented")


def refuse_data_parallel_debug(debug: bool, debug_from: int, world: int, who: str) -> None:
    if (debug or debug_from >= 0) and world > 1:
        raise ValueError(f"{who}: debug needs one GPU (world {world}): data-parallel debug mode is not implemented")


def renderer_set(rs, cls, model, P: int):
    """A trainer's evaluate() renderers: `rs` while it was made for the model's Gaussian count P, else a new set."""
    return rs if rs is not None and rs.P == P else RendererSet(cls, model, P)


def frame_for(frame, cam: Camera, max_size, make):
    """A trainer's frame for `cam`: made by make(W, H) at the first step, for max_size (default: the first view's size),
    and grown when a larger view arrives (_FrameSize.grow)."""
    W, H = int(cam.image_width), int(cam.image_height)
    if frame is None:
        frame = make(*(max_size or (W, H)))
    if W > frame.W or H > frame.H:
        frame.grow(W, H)
    return frame


class MeshTrainer:
    """fwd + loss + bwd (+ gradient all-reduce) + Adam for one frame per rank.

    fast=True  : fused expansion launch, packed SH features (zero-copy get_features), fused L1+SSIM loss kernels,
                 FlatAdam (one launch, zeroes the gradient) -- everything on the library's kernels except sigmoid.
    fast=False : the reference's op sequence (two-step expansion + getters, `loss_fn`, torch.optim.Adam) for A/B runs.

    Views may differ in size (one GPU): max_size (W, H), the largest view, sizes the one native frame (and the autograd
    arm's ground-truth buffer) once; without it they are sized from the first view and grow when a larger one arrives.

    antialiasing: the reference's pipe.antialiasing, a setting of the run: every training frame (native or autograd arm, one
    GPU or data parallel) and evaluate() render with it, and state_dict() records it.

    detect_anomaly: the reference's train.py --detect_anomaly (one GPU).  A native frame scans the outputs of each of its
    backward stages for NaN on the device and step() raises anomaly.AnomalyError, naming the first stage, tensor and element
    that held one, before before_update and before any parameter changes (the SH Adam step is not fused into the frame, one
    host synchronisation per step).  The autograd arm runs its step under torch.autograd.detect_anomaly().

    debug, debug_from: the reference's pipe.debug, train.py --debug and --debug_from (one GPU): debug mode from the first
    step, or from the step whose iteration - 1 == debug_from on.  A debug step copies what repeating it needs to the host
    (debug.DebugMode.snapshot), runs its frame with settings.debug and synchronises after every other library call; when it
    fails, the copy is written to `debug_snapshot`, the reference's message is printed, the trainer's state is put back and
    the error re-raised (debug.replay repeats the step)."""

    def __init__(self, model: MeshGaussianModel, bg: torch.Tensor, lambda_dssim: float = 0.2, world: int = 1,
                 rank: int = 0, optimizer_step: bool = True, fast: bool = True, native: bool = False, sync_free: bool = True,
                 loss_fn=None, sh_factored: bool = True, max_size: Optional[Tuple[int, int]] = None, antialiasing: bool = False,
                 detect_anomaly: bool = False, debug: bool = False, debug_from: int = -1, debug_snapshot: str = _debug.SNAPSHOT):
        refuse_data_parallel_anomaly(detect_anomaly, world, "MeshTrainer")
        refuse_data_parallel_debug(debug, debug_from, world, "MeshTrainer")
        if (debug or debug_from >= 0) and not (native and fast):
            raise ValueError("MeshTrainer: debug runs the native frame (native=True, fast=True); the autograd arms have no debug mode")
        self._debug = _debug.DebugMode(debug, debug_from, debug_snapshot)
        self.iteration = 0          # steps taken (debug_from counts them)
        self._sh_factored_arg = bool(sh_factored)
        self.model, self.bg, self.lambda_dssim = model, bg, lambda_dssim
        self.antialiasing = bool(antialiasing)
        self.detect_anomaly = bool(detect_anomaly)
        self._anomaly = None
        self.max_size = None if max_size is None else (int(max_size[0]), int(max_size[1]))
        self.world, self.rank = world, rank
        self.optimizer_step = optimizer_step
        self.fast = fast
        self.native = native and fast       # native: the whole frame is one C call (NativeFrame), no autograd
        self.sync_free = sync_free          # native frames after the first never synchronise with the host (NativeFrame)
        self.loss_fn = loss_fn or fused_training_loss    # fast=False A/B arm: callers may pass an ATen loss (tests/aten_reference.py)
        self._frame = None
        self._renderer = None
        self._gt_u8 = None      # the autograd arm's buffer for 8-bit ground truth
        self.sh_factored = False
        if fast:
            # native frames hand the SH gradient over as factors (12 B instead of 192 B per Gaussian; replicated optimizer);
            # the autograd-driven path materialises it (dense mode: sharded optimizer when world > 1)
            self.sh_factored = bool(sh_factored) and self.native and model._features is not None and model._features.shape[1] == 16
            self.opt = FlatAdam(mesh_model_groups(model, features_last=self.sh_factored), world=world, rank=rank, sh_factored=self.sh_factored)
            self.flat_grad = self.opt.flat_grad
        else:
            self.opt = model.training_setup()
            self.flat_grad = None

    def _all_reduce(self):
        if self.world <= 1:
            return
        if self.fast and self.optimizer_step:
            return      # FlatAdam.step() does reduce-scatter / sharded update / all-gather itself
        if self.flat_grad is not None:
            dist.all_reduce(self.flat_grad, op=dist.ReduceOp.SUM)
            self.flat_grad.mul_(1.0 / self.world)
        else:
            for p in self.model.parameters():
                if p.grad is not None:
                    dist.all_reduce(p.grad, op=dist.ReduceOp.SUM)
                    p.grad.mul_(1.0 / self.world)

    def _debug_config(self) -> dict:
        """The constructor arguments a replay (debug.replay) rebuilds this trainer with."""
        return dict(lambda_dssim=self.lambda_dssim, fast=self.fast, native=self.native, sync_free=self.sync_free,
                    sh_factored=self._sh_factored_arg, max_size=self.max_size, antialiasing=self.antialiasing)

    def _debug_flat(self) -> torch.Tensor:
        """The optimizer's flat parameter buffer (a debug snapshot takes the parameters from state_dict())."""
        return self.opt.p

    def _debug_restore(self, snap: dict) -> None:
        """The state a debug snapshot recorded before its step: parameters, moments, step counts, SH degree, iteration."""
        self.load_state_dict(_debug.to_device(snap["state_dict"], self.model.vertices.device))
        self.model.active_sh_degree = int(snap["active_sh_degree"])
        self.iteration = int(snap["iteration"]) - 1
        self.opt.zero_grad()

    @property
    def native_frame(self):
        """The native frame of the last step (None before the first)."""
        return self._frame

    def step(self, cam: Camera, gt: torch.Tensor, loss_host: Optional[torch.Tensor] = None,
             loss_ready: Optional[torch.cuda.Event] = None, bg: Optional[torch.Tensor] = None, before_update=None,
             frame_end: Optional[torch.cuda.Event] = None) -> torch.Tensor:
        """One optimisation step.  If `loss_host` (pinned) / `loss_ready` are given, the loss is copied to the host from a side
        stream as soon as the loss kernels have run (native frames: NativeFrame.read_loss_async; otherwise right after the
        backward pass, before the optimizer kernels are queued): a caller that logs the loss every step gets it while the
        backward pass is still running and queues its next step in that time.  gt: float32 [3,H,W] or uint8 [H,W,3].
        bg: this step's background instead of the trainer's (train.py's --random_background).  before_update: called after
        the frame and before any parameter changes (train.py's training_report and Scene.save see the parameters before the
        iteration's Adam step); the step then does not fuse the SH Adam update into the frame.  frame_end: recorded on the
        current stream right after the frame's launches (render, loss and backward, and on one GPU the SH Adam step the
        frame fuses in), before before_update and any other optimizer work: with an event recorded just before step(), it
        brackets train.py's iter_start / iter_end window.  In debug mode (debug, debug_from) the step runs as the class
        describes."""
        bg = self.bg if bg is None else bg
        it = self.iteration + 1
        loss = _debug.run_step(self, lambda debug: self._step(cam, gt, loss_host, loss_ready, bg, before_update, frame_end, debug),
                               cam, gt, bg, it)
        self.iteration = it
        return loss

    def _step(self, cam, gt, loss_host, loss_ready, bg, before_update, frame_end, debug: bool) -> torch.Tensor:
        if self.native:
            if self.world > 1:
                if self._frame is None:
                    self._frame = NativeFrame(self.model, cam.image_width, cam.image_height, self.lambda_dssim, sync_free=self.sync_free,
                                              world=self.world, rank=self.rank)
                elif (int(cam.image_width), int(cam.image_height)) != (self._frame.W, self._frame.H):
                    raise ValueError(f"MeshTrainer: data-parallel training (world {self.world}) needs every view at one size, "
                                     f"{self._frame.W}x{self._frame.H}; got a {cam.image_width}x{cam.image_height} camera: "
                                     f"views of mixed sizes are trained on one GPU only")
            else:
                self._frame = frame_for(self._frame, cam, self.max_size, lambda W, H: NativeFrame(
                    self.model, W, H, self.lambda_dssim, sync_free=self.sync_free, up_to=True))
            factored = self.sh_factored and self.optimizer_step      # without an optimizer step the full gradient is materialised
            # one GPU: the frame applies the SH Adam step itself (no colour-gradient slot, no second read of the SH rows);
            # data parallel: the colour gradients are exchanged first and k_adam_sh consumes them
            fused = factored and self.world == 1 and before_update is None and not self.detect_anomaly
            sh_adam = self.opt.begin_fused_sh_step() if fused else None
            record = anomaly_record(self._anomaly, self._frame.dev) if self.detect_anomaly else None
            self._anomaly = record
            loss = self._frame.run(cam, gt, bg, factored=factored and not fused, sh_adam=sh_adam, antialiasing=self.antialiasing,
                                   anomaly=record, debug=debug)
            if frame_end is not None:
                frame_end.record(torch.cuda.current_stream(self._frame.dev))
            from . import rasterizer as _r
            _r.last_num_rendered = self._frame.last_num_rendered
            if loss_host is not None:
                self._frame.read_loss_async(loss_host, loss_ready)
            if record is not None:
                check_anomaly(record, self.model, cam, self.opt)
            if before_update is not None:
                before_update()
            self._all_reduce()
            # gms_train_frame overwrites every gradient except the atomically accumulated vertex segment (group 0)
            if fused:
                self.opt.step_rest(zero_end=self.opt.ends[0])
            elif self.optimizer_step:
                self.opt.step(zero_end=self.opt.ends[0], sh=self._frame.sh_factors() if factored else None)
            else:
                self.opt.zero_grad_partial(self.opt.ends[0])
            if debug:
                _debug.sync("FlatAdam step (gms_adam_step, gms_adam_sh_factored)", self._frame.dev)
            return loss
        if gt.dtype == torch.uint8:
            H, W = int(gt.shape[0]), int(gt.shape[1])
            b = self._gt_u8
            if b is None or H > b.H or W > b.W:         # sized for max_size (and any earlier view), grown for a larger view
                mW, mH = self.max_size or (0, 0)
                self._gt_u8 = GroundTruthBuffer(max(H, mH, b.H if b else 0), max(W, mW, b.W if b else 0), self.model.vertices.device,
                                                up_to=True)
            gt = self._gt_u8(gt, "MeshTrainer.step")
        from . import rasterizer as _r
        prev = _r.DIRECT_SH_GRAD
        _r.DIRECT_SH_GRAD = self.fast      # FlatAdam keeps .grad preallocated and zeroed: write dL/dshs in place
        try:
            with torch.autograd.detect_anomaly() if self.detect_anomaly else contextlib.nullcontext():
                image, radii, _ = render_frame(self.model, cam, bg, fused=self.fast, antialiasing=self.antialiasing)
                loss = fused_training_loss(image, gt, self.lambda_dssim) if self.fast else self.loss_fn(image, gt, self.lambda_dssim)
                loss.backward()
        finally:
            _r.DIRECT_SH_GRAD = prev       # never leak the in-place mode to other users of the rasterizer
        if frame_end is not None:
            frame_end.record(torch.cuda.current_stream(loss.device))
        if loss_host is not None:
            loss_host.copy_(loss.detach().reshape(loss_host.shape), non_blocking=True)
            if loss_ready is not None:
                loss_ready.record(torch.cuda.current_stream(loss.device))
        if before_update is not None:
            before_update()
        self._all_reduce()
        if self.optimizer_step:
            self.opt.step()
            if not self.fast:
                self.opt.zero_grad(set_to_none=False)
        elif self.fast:
            self.opt.zero_grad()
        else:
            for p in self.model.parameters():
                p.grad = None
        return loss.detach()

    @property
    def renderer(self):
        """The renderers (render.RendererSet) the last evaluate() built or reused, one per image size, sized for the
        model's current Gaussian count (None before the first): renderer.render(cam, bg) draws a view of the current model
        at the view's size without a second copy of the model."""
        return self._renderer

    def evaluate(self, cams: Sequence[Camera], gts: Sequence[torch.Tensor], protocol: str = "training_report"):
        """L1 / SSIM / PSNR of the current model on held-out views with the trainer's background, the test half of
        training_report (train.py:183-218): NativeRenderer.evaluate, one host synchronisation per image size of the set."""
        self._renderer = renderer_set(self._renderer, NativeRenderer, self.model, self.model._scale.shape[0])
        return self._renderer.evaluate(cams, gts, self.bg, protocol=protocol, antialiasing=self.antialiasing, debug=self._debug.on)

    def state_dict(self) -> dict:
        """What resuming needs (single GPU, fast=True): FlatAdam's flat parameters, moments and step counts, the active SH
        degree and the antialiasing setting.  Copies on the device."""
        if not self.fast:
            raise ValueError("MeshTrainer.state_dict needs the FlatAdam trainer (fast=True)")
        return {"adam": self.opt.state_dict(), "active_sh_degree": int(self.model.active_sh_degree), "antialiasing": self.antialiasing}

    def load_state_dict(self, state: dict) -> None:
        """Restores state_dict(); refuses a state trained with the other antialiasing setting."""
        if not self.fast:
            raise ValueError("MeshTrainer.load_state_dict needs the FlatAdam trainer (fast=True)")
        check_antialiasing(state, self.antialiasing, "MeshTrainer")
        self.opt.load_state_dict(state["adam"])
        self.model.active_sh_degree = int(state["active_sh_degree"])
        self.iteration = self.opt.t


# ---------------------------------------------------------------------------------------------- free Gaussians (gs, gs_flat)

@dataclass
class FreeOptimizationParams:
    """OptimizationParams of the reference (arguments/__init__.py:72-91) that a gs / gs_flat run reads."""
    iterations: int = 30_000
    position_lr_init: float = 0.00016
    position_lr_final: float = 0.0000016
    position_lr_delay_mult: float = 0.01
    position_lr_max_steps: int = 30_000
    feature_lr: float = 0.0025
    opacity_lr: float = 0.05
    scaling_lr: float = 0.005
    rotation_lr: float = 0.001
    percent_dense: float = 0.01
    lambda_dssim: float = 0.2
    densification_interval: int = 100
    opacity_reset_interval: int = 3000
    densify_from_iter: int = 500
    densify_until_iter: int = 15_000
    densify_grad_threshold: float = 0.0002
    min_opacity: float = 0.005          # densify_and_prune's second argument (train.py:143)


def expon_lr(step: int, lr_init: float, lr_final: float, lr_delay_steps: int = 0, lr_delay_mult: float = 1.0,
             max_steps: int = 1_000_000) -> float:
    """get_expon_lr_func (utils/general_utils.py:109-145) evaluated at `step`."""
    if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
        return 0.0
    delay = lr_delay_mult + (1 - lr_delay_mult) * np.sin(0.5 * np.pi * np.clip(step / lr_delay_steps, 0, 1)) if lr_delay_steps > 0 else 1.0
    t = np.clip(step / max_steps, 0, 1)
    return float(delay * np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t))


class NativeFreeFrame(_FrameSize):
    """One gs / gs_flat training frame through gms_free_train_frame: activation, rasterizer, loss, backward and (optionally)
    the densification statistics in ONE C call.  Gradients land in the parameters' .grad views (FlatAdam's flat buffer).

    Sync-free like NativeFrame, with one addition: after the model's Gaussian count changed (resize()), every view's next
    frame learns its N with one read-back, so a growing model loses no frame to an overflowed capacity.

    up_to: width x height is the largest view; smaller views run at their own size in the same workspace (_FrameSize)."""

    def __init__(self, model, width: int, height: int, lambda_dssim: float = 0.2, sync_free: bool = True, up_to: bool = False):
        self.model, self.lam = model, float(lambda_dssim)
        self.dev = model._xyz.device
        self.loss = torch.zeros(3, dtype=torch.float32, device=self.dev)
        self._init_capacity(sync_free)
        self._scratch, self._cb = grow_only_alloc(self.dev)
        self.ws = None
        self.ev_loss = None
        self._init_size(width, height, up_to)
        self.resize()

    def _gaussians(self) -> int:
        return self.model.P

    def resize(self) -> None:
        """The model's P changed: grow the workspace (for the frame's largest view), zero the statistics, forget every
        view's N."""
        P = self.model.P
        self._fit_workspace()
        self.accum = torch.zeros(P, dtype=torch.float32, device=self.dev)
        self.denom = torch.zeros(P, dtype=torch.float32, device=self.dev)
        self._forget_views()

    def _check(self, gt, bg, cam):
        m = self.model
        for n in m.NAMES:
            t = getattr(m, n)
            check_float32(t, f"NativeFreeFrame: model.{n}", self.dev)
            if t.grad is None or not t.grad.is_contiguous() or t.grad.shape != t.shape:
                raise RuntimeError(f"NativeFreeFrame: model.{n}.grad must be a preallocated contiguous buffer (FlatAdam provides it)")
        if self.accum.shape[0] != m.P:
            raise RuntimeError("NativeFreeFrame: the model's Gaussian count changed; call resize()")
        self._check_view(cam, bg, "NativeFreeFrame.run", gt=gt, gt_fits=lambda W, H: tuple(gt.shape) == (3, H, W))

    def run(self, cam: Camera, gt: torch.Tensor, bg: torch.Tensor, stats: bool = True, sh_adam=None,
            antialiasing: bool = False, anomaly: Optional[AnomalyRecord] = None, anomaly_stages: int = FRAME_STAGES,
            debug: bool = False) -> torch.Tensor:
        """stats: add this frame's densification statistics to `accum` / `denom`.  sh_adam (FlatAdam.begin_fused_sh_step()):
        the frame also applies the SH parameters' Adam step and writes no SH gradient.  gt: float32 [3,H,W], or uint8 [H,W,3]
        (dequantized on the device into the frame's buffer).  antialiasing, anomaly, anomaly_stages, debug: as NativeFrame.run."""
        import ctypes as C
        from . import _lib
        if gt.dtype == torch.uint8:
            gt = self._gt_u8(gt, "NativeFreeFrame.run")
            if debug:
                _debug.sync("gms_image_dequantize", self.dev)
        gt = gt.contiguous()
        self._check(gt, bg, cam)
        m = self.model
        a = _lib.FreeFrameArgs()
        a.P, a.M, a.scale_cols = m.P, m._features.shape[1], m.scale_cols
        a.xyz, a.scaling_raw, a.rotation_raw = m._xyz.data_ptr(), m._scaling.data_ptr(), m._rotation.data_ptr()
        a.features, a.opacity_raw, a.eps = m._features.data_ptr(), m._opacity.data_ptr(), m.eps_s0
        a.d_xyz, a.d_scaling_raw, a.d_rotation_raw = m._xyz.grad.data_ptr(), m._scaling.grad.data_ptr(), m._rotation.grad.data_ptr()
        a.d_features, a.d_opacity_raw = m._features.grad.data_ptr(), m._opacity.grad.data_ptr()
        if sh_adam is not None:
            a.d_features, a.sh_adam = None, C.pointer(sh_adam)
        if stats:
            a.accum, a.denom = self.accum.data_ptr(), self.denom.data_ptr()
        self.ev_loss = recorded_event(self.ev_loss, self.dev)
        a.event_loss_ready = self.ev_loss.cuda_event
        a.gt, a.lambda_dssim, a.loss = gt.data_ptr(), self.lam, self.loss.data_ptr()
        if anomaly is not None:
            a.anomaly, a.anomaly_stages = anomaly.ptr, int(anomaly_stages)
        self._launch("gms_free_train_frame", a, cam, bg, antialiasing=antialiasing, **({"debug": True} if debug else {}))
        return self.loss[0]


def densify_plan(model, accum, denom, extent: float, opt: FreeOptimizationParams, size_prune: bool):
    """gms_densify_plan on the model's current rows: (result [new P, kept, clones, split pairs, pruned], fate [P] uint8,
    scratch).  One host synchronisation."""
    import ctypes as C
    from . import _lib
    P = model.P
    scratch = torch.empty(int(_lib.lib().gms_densify_scratch_bytes(P)), dtype=torch.uint8, device=model._xyz.device)
    fate = torch.empty(max(P, 1), dtype=torch.uint8, device=model._xyz.device)
    res = (C.c_int32 * 5)()
    a = _lib.DensifyPlanArgs()
    a.P, a.scale_cols = P, model.scale_cols
    a.accum, a.denom, a.scaling_raw, a.opacity_raw = accum.data_ptr(), denom.data_ptr(), model._scaling.data_ptr(), model._opacity.data_ptr()
    a.eps, a.grad_threshold = model.eps_s0, opt.densify_grad_threshold
    a.split_scale, a.min_opacity = opt.percent_dense * extent, opt.min_opacity
    a.max_world_scale = 0.1 * extent if size_prune else 0.0
    a.fate, a.scratch, a.scratch_bytes, a.result = fate.data_ptr(), scratch.data_ptr(), scratch.numel(), res
    with torch.cuda.device(model._xyz.device):
        _lib.check(_lib.lib().gms_densify_plan(C.byref(a), torch.cuda.current_stream(model._xyz.device).cuda_stream), "gms_densify_plan")
    return list(res), fate[:P], scratch


def densify_apply(model, plan, normals, old: dict, new: dict) -> None:
    """gms_densify_apply: `old` / `new` map "p", "m", "v" to per-tensor lists in FreeGaussianModel.NAMES order."""
    import ctypes as C
    from . import _lib
    res, _, scratch = plan
    a = _lib.DensifyApplyArgs()
    a.P, a.new_P, a.scale_cols, a.M, a.eps = model.P, res[0], model.scale_cols, model._features.shape[1], model.eps_s0
    a.scratch, a.scratch_bytes, a.result = scratch.data_ptr(), scratch.numel(), (C.c_int32 * 5)(*res)
    a.normals = normals.data_ptr()
    for t, k in enumerate(("p", "m", "v")):
        for dst, src in ((a.dst[t], new[k]), (a.src[t], old[k])):
            dst.xyz, dst.scaling, dst.rotation, dst.opacity, dst.features = (x.data_ptr() for x in src)
    with torch.cuda.device(model._xyz.device):
        _lib.check(_lib.lib().gms_densify_apply(C.byref(a), torch.cuda.current_stream(model._xyz.device).cuda_stream), "gms_densify_apply")


class FreeTrainer:
    """A whole iteration of the reference's train.py:83-157 for gs / gs_flat, on one GPU:

        update_learning_rate (xyz schedule) -> oneupSHdegree every 1000 -> gms_free_train_frame with the densification
        statistics -> densify_and_prune / reset_opacity at the reference's schedule -> Adam.

    Reproduced quirks of the reference:
      - max_radii2D is not tracked: densification_postfix zeroes it on every densify_and_prune before it is read, so the
        screen-size prune never fires; only the world-size prune (max scale > 0.1 * extent, after opacity_reset_interval) does.
      - On a densification iteration every parameter is replaced by one without a gradient, so optimizer.step() updates
        nothing and no step count advances; the frame then runs without the fused SH step.  A lone opacity reset (white
        background at densify_from_iter) skips the opacity group only, whose bias correction lags by one from then on.
      - Appended rows start with zero Adam moments; reset_opacity zeroes the opacity moments.
    The split samples come from torch.randn on the device (`generator`).  Views may differ in size: max_size (W, H) as
    MeshTrainer's; the frame keeps its size when densification changes P.  antialiasing: as MeshTrainer's.  detect_anomaly: as
    MeshTrainer's; step() raises before densification, the opacity reset and Adam, with the iteration counter and the
    densification statistics as they were before the step (the learning rate and SH degree of the iteration stay applied, as
    in the reference).  debug, debug_from, debug_snapshot: as MeshTrainer's; a failed debug step leaves the iteration
    counter, the densification statistics and the split generator as they were before it."""

    def __init__(self, model, bg: torch.Tensor, extent: float, opt: FreeOptimizationParams = None, white_background: bool = None,
                 sync_free: bool = True, world: int = 1, generator: torch.Generator = None,
                 max_size: Optional[Tuple[int, int]] = None, antialiasing: bool = False, detect_anomaly: bool = False,
                 debug: bool = False, debug_from: int = -1, debug_snapshot: str = _debug.SNAPSHOT):
        refuse_data_parallel_anomaly(detect_anomaly, world, "FreeTrainer")
        refuse_data_parallel_debug(debug, debug_from, world, "FreeTrainer")
        self._debug = _debug.DebugMode(debug, debug_from, debug_snapshot)
        if world != 1:
            raise ValueError("FreeTrainer trains on one GPU: data-parallel densification (all-reduced statistics) is not implemented")
        from .optim import free_model_groups
        self.model, self.bg, self.extent = model, bg, float(extent)
        self.opt = opt or FreeOptimizationParams()
        self.white_background = bool((bg == 1).all()) if white_background is None else bool(white_background)
        self.sync_free, self.generator = sync_free, generator
        self.max_size = None if max_size is None else (int(max_size[0]), int(max_size[1]))
        self.antialiasing = bool(antialiasing)
        self.detect_anomaly = bool(detect_anomaly)
        self._anomaly = None
        o = self.opt
        self.fused_sh = model._features.shape[1] == 16
        self.adam = FlatAdam(free_model_groups(model, self._xyz_lr(0), o.feature_lr, o.opacity_lr, o.scaling_lr, o.rotation_lr),
                             sh_factored=self.fused_sh)
        self.iteration = 0
        self.frame = None
        self._renderer = None
        self._loaded_stats = None       # (accum, denom) of load_state_dict, until the first frame exists
        self.densifications = []        # (iteration, P before, result of the plan)

    def _xyz_lr(self, it: int) -> float:
        o = self.opt
        return expon_lr(it, o.position_lr_init * self.extent, o.position_lr_final * self.extent, lr_delay_mult=o.position_lr_delay_mult,
                        max_steps=o.position_lr_max_steps)

    def schedule(self, it: int):
        """(statistics, densify, reset_opacity) of iteration `it` (1-based), train.py:133-149."""
        o = self.opt
        if it >= o.densify_until_iter:
            return False, False, False
        densify = it > o.densify_from_iter and it % o.densification_interval == 0
        reset = it % o.opacity_reset_interval == 0 or (self.white_background and it == o.densify_from_iter)
        return True, densify, reset

    @property
    def loss_vector(self) -> Optional[torch.Tensor]:
        """The frame's device [3] vector [loss, L1, SSIM] of the last step (None before the first): the next step overwrites
        it in stream order."""
        return None if self.frame is None else self.frame.loss

    def step(self, cam: Camera, gt: torch.Tensor, bg: torch.Tensor = None, before_update=None,
             frame_end: Optional[torch.cuda.Event] = None) -> torch.Tensor:
        """One iteration.  bg: this step's background instead of the trainer's (train.py's --random_background).
        before_update: called after the frame and before densify / opacity reset / Adam (train.py's training_report and
        Scene.save see the parameters before the iteration's update); the step then does not fuse the SH Adam update into
        the frame.  frame_end: recorded on the current stream right after the frame's launches, before before_update,
        densification and any Adam step outside the frame (MeshTrainer.step)."""
        it = self.iteration + 1
        bg = self.bg if bg is None else bg
        return _debug.run_step(self, lambda debug: self._step(cam, gt, bg, before_update, frame_end, debug), cam, gt, bg, it)

    def _debug_config(self) -> dict:
        """The constructor arguments a replay (debug.replay) rebuilds this trainer with."""
        return dict(extent=self.extent, opt=self.opt, white_background=self.white_background, sync_free=self.sync_free,
                    max_size=self.max_size, antialiasing=self.antialiasing)

    def _debug_flat(self) -> torch.Tensor:
        return self.adam.p

    def _debug_restore(self, snap: dict) -> None:
        """The state a debug snapshot recorded before its step (MeshTrainer._debug_restore), statistics and generator too."""
        self.load_state_dict(_debug.to_device(snap["state_dict"], self.model._xyz.device))
        self.model.active_sh_degree = int(snap["active_sh_degree"])
        self.iteration = int(snap["iteration"]) - 1
        self.adam.zero_grad()

    @property
    def native_frame(self):
        """The native frame of the last step (None before the first)."""
        return self.frame

    def _step(self, cam, gt, bg, before_update, frame_end, debug: bool) -> torch.Tensor:
        it = self.iteration + 1
        self.adam.groups[0]["lr"] = self._xyz_lr(it)
        if it % 1000 == 0:
            self.model.oneupSHdegree()
        stats, densify, reset = self.schedule(it)
        self.frame = frame_for(self.frame, cam, self.max_size, lambda W, H: NativeFreeFrame(
            self.model, W, H, self.opt.lambda_dssim, sync_free=self.sync_free, up_to=True))
        if self._loaded_stats is not None:      # load_state_dict before the first frame existed
            self.frame.accum.copy_(self._loaded_stats[0])
            self.frame.denom.copy_(self._loaded_stats[1])
            self._loaded_stats = None
        fuse = self.fused_sh and not densify and before_update is None and not self.detect_anomaly
        sh_adam = self.adam.begin_fused_sh_step() if fuse else None
        record, restore = None, None
        if self.detect_anomaly:
            record = self._anomaly = anomaly_record(self._anomaly, self.frame.dev)
            if stats:       # the frame adds this step's statistics in its last kernel
                f, kept = self.frame, (self.frame.accum.clone(), self.frame.denom.clone())
                restore = lambda: (f.accum.copy_(kept[0]), f.denom.copy_(kept[1]))
        loss = self.frame.run(cam, gt, bg, stats=stats, sh_adam=sh_adam, antialiasing=self.antialiasing, anomaly=record, debug=debug)
        if frame_end is not None:
            frame_end.record(torch.cuda.current_stream(self.frame.dev))
        if record is not None:
            check_anomaly(record, self.model, cam, self.adam, it, restore)
        if before_update is not None:
            before_update()
        if densify:
            self.densify(size_prune=it > self.opt.opacity_reset_interval)
            if debug:
                _debug.sync("densification (gms_densify_plan, gms_densify_apply)", self.frame.dev)
        if reset:
            self.reset_opacity()
        if not densify and it < self.opt.iterations:     # train.py steps the optimizer on every iteration but the last
            skip = ("opacity",) if reset else ()
            if sh_adam is not None:
                self.adam.step_rest(zero_end=0, skip=skip)
            elif self.fused_sh:
                self.adam.step_dense(zero_end=0, skip=skip)
            else:
                self.adam.step(zero_end=0, skip=skip)
            if debug:
                _debug.sync("FlatAdam step (gms_adam_step)", self.frame.dev)
        self.iteration = it
        return loss

    def state_dict(self) -> dict:
        """What resuming needs: FlatAdam's flat parameters, moments, group shapes and step counts, the active SH degree, the
        iteration, P, the frame's densification statistics, the split generator's state and the antialiasing setting.  Copies
        on the device."""
        dev = self.model._xyz.device
        f = self.frame
        if f is not None:
            accum, denom = f.accum.detach().clone(), f.denom.detach().clone()
        elif self._loaded_stats is not None:
            accum, denom = (t.detach().clone() for t in self._loaded_stats)
        else:
            accum = torch.zeros(self.model.P, dtype=torch.float32, device=dev)
            denom = torch.zeros(self.model.P, dtype=torch.float32, device=dev)
        gen = self.generator.get_state() if self.generator is not None else torch.cuda.get_rng_state(dev)
        return {"adam": self.adam.state_dict(), "active_sh_degree": int(self.model.active_sh_degree), "iteration": int(self.iteration),
                "P": int(self.model.P), "accum": accum, "denom": denom, "generator": gen, "antialiasing": self.antialiasing}

    def load_state_dict(self, state: dict) -> None:
        """Restores state_dict(), also when the state's P differs from the model's (densified before it was captured); refuses
        a state trained with the other antialiasing setting."""
        dev = self.model._xyz.device
        check_antialiasing(state, self.antialiasing, "FreeTrainer")
        self.adam.load_state_dict(state["adam"])
        if self.model.P != int(state["P"]):
            raise ValueError(f"FreeTrainer.load_state_dict: the state holds P = {state['P']} but its parameters {self.model.P}")
        self.model.active_sh_degree = int(state["active_sh_degree"])
        self.iteration = int(state["iteration"])
        accum, denom = state["accum"].to(dev), state["denom"].to(dev)
        if self.frame is not None:
            self.frame.resize()
            self.frame.accum.copy_(accum)
            self.frame.denom.copy_(denom)
        else:
            self._loaded_stats = (accum, denom)
        if self.generator is not None:
            self.generator.set_state(state["generator"].cpu())
        else:
            torch.cuda.set_rng_state(state["generator"].cpu(), dev)

    def densify(self, size_prune: bool, normals: torch.Tensor = None) -> list:
        """densify_and_prune(densify_grad_threshold, min_opacity, extent, 20 if size_prune else None) on the statistics
        gathered so far; the frame's gradients are discarded.  normals [P,2,3]: the split draws (default torch.randn)."""
        m, f = self.model, self.frame
        P0 = m.P
        plan = densify_plan(m, f.accum, f.denom, self.extent, self.opt, size_prune)
        if normals is None:
            normals = torch.randn(max(P0, 1), 2, 3, device=m._xyz.device, generator=self.generator)
        newP = plan[0][0]
        names = [g["name"] for g in self.adam.groups]
        tensor_of = {"xyz": "_xyz", "opacity": "_opacity", "scaling": "_scaling", "rotation": "_rotation", "features": "_features"}
        order = [names.index(k) for k in ("xyz", "scaling", "rotation", "opacity", "features")]     # FreeGaussianModel.NAMES order

        def fill(old, new):
            densify_apply(m, plan, normals, {k: [old[k][i] for i in order] for k in old}, {k: [new[k][i] for i in order] for k in new})

        self.adam.resize([(newP,) + tuple(getattr(m, tensor_of[n]).shape[1:]) for n in names], fill)
        f.resize()
        self.densifications.append((self.iteration + 1, P0, plan[0]))
        return plan[0]

    def reset_opacity(self) -> None:
        """reset_opacity (scene/gaussian_model.py:218-221) on the flat views: opacity = inverse_sigmoid(min(sigmoid, 0.01)),
        opacity moments zeroed."""
        i = self.adam.group_index("opacity")
        op = self.model._opacity.data
        x = torch.min(torch.sigmoid(op), torch.ones_like(op) * 0.01)
        op.copy_(torch.log(x / (1 - x)))
        o0, o1 = (self.adam.ends[i - 1] if i else 0), self.adam.ends[i]
        self.adam.m[o0:o1].zero_()
        self.adam.v[o0:o1].zero_()

    @property
    def renderer(self):
        """The renderer the last evaluate() built or reused (MeshTrainer.renderer)."""
        return self._renderer

    def evaluate(self, cams: Sequence[Camera], gts: Sequence[torch.Tensor], protocol: str = "training_report"):
        """L1 / SSIM / PSNR of the current model on held-out views (NativeFreeRenderer.evaluate, MeshTrainer.evaluate)."""
        self._renderer = renderer_set(self._renderer, NativeFreeRenderer, self.model, self.model.P)
        return self._renderer.evaluate(cams, gts, self.bg, protocol=protocol, antialiasing=self.antialiasing, debug=self._debug.on)


# ---------------------------------------------------------------------------------------------- gs_flame

@dataclass
class FlameOptimizationParams:
    """OptimizationParamsFlame of the reference (arguments_games/__init__.py:32-49)."""
    iterations: int = 30_000
    alpha_lr: float = 0.001
    feature_lr: float = 0.0025
    opacity_lr: float = 0.05
    scaling_lr: float = 0.005
    flame_shape_lr: float = 0.01
    flame_exp_lr: float = 0.001
    flame_pose_lr: float = 0.001
    flame_neck_pose_lr: float = 0.001
    flame_trans_lr: float = 0.001
    vertices_enlargement_lr: float = 0.0002
    lambda_dssim: float = 0.2


def flame_model_groups(model, o: FlameOptimizationParams) -> List[dict]:
    """GaussianFlameModel.training_setup's groups (gaussian_flame_model.py:209-224) in its order, f_dc / f_rest as the one
    packed SH group moved to the end (what FlatAdam(sh_factored=True) needs; the order of Adam groups has no numerical
    meaning)."""
    M = model._features.shape[1]
    return [dict(param=model._flame_shape, lr=o.flame_shape_lr, name="shape"),
            dict(param=model._flame_exp, lr=o.flame_exp_lr, name="expression"),
            dict(param=model._flame_pose, lr=o.flame_pose_lr, name="pose"),
            dict(param=model._flame_neck_pose, lr=o.flame_neck_pose_lr, name="neck_pose"),
            dict(param=model._flame_trans, lr=o.flame_trans_lr, name="transl"),
            dict(param=model._vertices_enlargement, lr=o.vertices_enlargement_lr, name="vertices_enlargement"),
            dict(param=model._alpha, lr=o.alpha_lr, name="alpha"),
            dict(param=model._opacity, lr=o.opacity_lr, name="opacity"),
            dict(param=model._scales, lr=o.scaling_lr, name="scaling"),
            dict(param=model._features, lr0=o.feature_lr, lr1=o.feature_lr / 20.0, inner=3, period=M, name="features")]


class FlameTrainer:
    """A whole iteration of the reference's train.py:83-157 for gs_flame (FlameGaussianModel), on one GPU:

        oneupSHdegree every 1000 -> the driver's forward (ATen, autograd graph kept) -> gms_train_frame with softmax
        weights on the detached vertices -> dL/dvertices back through the driver (torch.autograd.backward) -> Adam over the
        reference's groups (FlatAdam; the SH step fused into the frame when M = 16).

    With a NativeFlame driver there is no autograd graph: gms_flame_lbs_forward writes model.vertices, and
    gms_flame_lbs_backward writes the FLAME gradients into FlatAdam's slots (no host synchronisation after the first step).

    No densification (train.py densifies gs / gs_flat only), a constant learning rate per group (update_learning_rate is a
    no-op, gaussian_flame_model.py:226-228), and no optimizer step at the last iteration.  After step(), model.vertices
    holds the pose the step rendered, not the updated parameters' (model.refresh_vertices() moves it; evaluate() does).
    Views may differ in size: max_size (W, H) as MeshTrainer's.  antialiasing: as MeshTrainer's.  detect_anomaly: as
    MeshTrainer's, with the iteration counter unchanged when step() raises; a NativeFlame driver's parameter gradients are
    scanned as one more stage (FLAME backward), and the ATen part of any other driver runs under
    torch.autograd.detect_anomaly() after the frame's record was read.  debug, debug_from, debug_snapshot: as MeshTrainer's;
    a debug step also synchronises after the NativeFlame LBS forward and backward."""

    def __init__(self, model, bg: torch.Tensor, opt: FlameOptimizationParams = None, sync_free: bool = True,
                 max_size: Optional[Tuple[int, int]] = None, antialiasing: bool = False, detect_anomaly: bool = False,
                 debug: bool = False, debug_from: int = -1, debug_snapshot: str = _debug.SNAPSHOT):
        self._debug = _debug.DebugMode(debug, debug_from, debug_snapshot)
        self.model, self.bg = model, bg
        self.antialiasing = bool(antialiasing)
        self.detect_anomaly = bool(detect_anomaly)
        self._anomaly = None
        self.max_size = None if max_size is None else (int(max_size[0]), int(max_size[1]))
        self.opt = opt or FlameOptimizationParams()
        self.sync_free = sync_free
        self.fused_sh = model._features.shape[1] == 16
        self.adam = FlatAdam(flame_model_groups(model, self.opt), sh_factored=self.fused_sh)
        self.iteration = 0
        self.frame = None
        self._renderer = None
        self._lbs = None

    @property
    def loss_vector(self) -> Optional[torch.Tensor]:
        """The frame's device [3] vector [loss, L1, SSIM] of the last step (None before the first): the next step overwrites
        it in stream order."""
        return None if self.frame is None else self.frame.loss

    def step(self, cam: Camera, gt: torch.Tensor, bg: Optional[torch.Tensor] = None, before_update=None,
             frame_end: Optional[torch.cuda.Event] = None) -> torch.Tensor:
        """One iteration.  bg: this step's background instead of the trainer's (train.py's --random_background).
        before_update: called after the frame and the driver's backward, before any parameter changes (train.py's
        training_report and Scene.save see the parameters before the iteration's Adam step); the step then does not fuse the
        SH Adam update into the frame.  frame_end: recorded on the current stream right after the frame's launches and the
        driver's backward, before before_update and any Adam step outside the frame (MeshTrainer.step)."""
        it = self.iteration + 1
        bg = self.bg if bg is None else bg
        return _debug.run_step(self, lambda debug: self._step(cam, gt, bg, before_update, frame_end, debug), cam, gt, bg, it)

    def _debug_config(self) -> dict:
        """The constructor arguments a replay (debug.replay) rebuilds this trainer with."""
        return dict(opt=self.opt, sync_free=self.sync_free, max_size=self.max_size, antialiasing=self.antialiasing)

    def _debug_flat(self) -> torch.Tensor:
        return self.adam.p

    def _debug_restore(self, snap: dict) -> None:
        """The state a debug snapshot recorded before its step (MeshTrainer._debug_restore)."""
        self.load_state_dict(_debug.to_device(snap["state_dict"], self.model.vertices.device))
        self.model.active_sh_degree = int(snap["active_sh_degree"])
        self.iteration = int(snap["iteration"]) - 1
        self.adam.zero_grad()

    @property
    def native_frame(self):
        """The native frame of the last step (None before the first)."""
        return self.frame

    def _step(self, cam, gt, bg, before_update, frame_end, debug: bool) -> torch.Tensor:
        it = self.iteration + 1
        m = self.model
        if it % 1000 == 0:
            m.oneupSHdegree()
        native = isinstance(m.driver, NativeFlame)
        aten_anomaly = lambda: torch.autograd.detect_anomaly() if self.detect_anomaly else contextlib.nullcontext()
        if native:
            if self._lbs is None:
                self._lbs = m.driver.bind(m)
            self._lbs.forward()                  # into model.vertices; zeroes model.vertices.grad
            if debug:
                _debug.sync("gms_flame_lbs_forward", self.model.vertices.device)
        else:
            with aten_anomaly():
                verts = m.driver_vertices()
            with torch.no_grad():
                m.vertices.copy_(verts)
            m.vertices.grad.zero_()
        self.frame = frame_for(self.frame, cam, self.max_size, lambda W, H: NativeFrame(
            m, W, H, self.opt.lambda_dssim, sync_free=self.sync_free, up_to=True))
        take_step = it < self.opt.iterations         # train.py steps the optimizer on every iteration but the last
        fused = self.fused_sh and take_step and before_update is None and not self.detect_anomaly
        sh_adam = self.adam.begin_fused_sh_step() if fused else None
        record = anomaly_record(self._anomaly, self.frame.dev) if self.detect_anomaly else None
        self._anomaly = record
        loss = self.frame.run(cam, gt, bg, sh_adam=sh_adam, antialiasing=self.antialiasing, anomaly=record, debug=debug)
        if native:
            self._lbs.backward()                 # writes the FLAME tensors' flat .grad views
            if debug:
                _debug.sync("gms_flame_lbs_backward", self.frame.dev)
            if record is not None:
                record.scan(_lib.ANOMALY_FLAME_BWD, [(i, getattr(m, n).grad) for i, n in enumerate(m.FLAME_NAMES)])
                check_anomaly(record, m, cam, self.adam, it)
        else:
            if record is not None:               # the frame's stages come first, as in one autograd backward
                check_anomaly(record, m, cam, self.adam, it)
            with aten_anomaly():
                torch.autograd.backward(verts, m.vertices.grad)      # accumulates into the FLAME tensors' flat .grad views
        if frame_end is not None:
            frame_end.record(torch.cuda.current_stream(self.frame.dev))
        if before_update is not None:
            before_update()
        if not take_step:
            self.adam.zero_grad()
        elif fused:
            self.adam.step_rest()
        elif self.fused_sh:
            self.adam.step_dense()
        else:
            self.adam.step()
        if debug:
            _debug.sync("FlatAdam step (gms_adam_step)", self.frame.dev)
        self.iteration = it
        return loss

    def state_dict(self) -> dict:
        """What resuming needs: FlatAdam's flat parameters (the FLAME tensors among them), moments and step counts, the active
        SH degree, the iteration and the antialiasing setting.  Copies on the device."""
        return {"adam": self.adam.state_dict(), "active_sh_degree": int(self.model.active_sh_degree), "iteration": int(self.iteration),
                "antialiasing": self.antialiasing}

    def load_state_dict(self, state: dict) -> None:
        """Restores state_dict(); refuses a state trained with the other antialiasing setting."""
        check_antialiasing(state, self.antialiasing, "FlameTrainer")
        self.adam.load_state_dict(state["adam"])
        self.model.active_sh_degree = int(state["active_sh_degree"])
        self.iteration = int(state["iteration"])

    @property
    def renderer(self):
        """The renderer the last evaluate() built or reused (MeshTrainer.renderer)."""
        return self._renderer

    def evaluate(self, cams: Sequence[Camera], gts: Sequence[torch.Tensor], protocol: str = "training_report"):
        """L1 / SSIM / PSNR of the current model (at its current pose) on held-out views (MeshTrainer.evaluate)."""
        self.model.refresh_vertices()
        self._renderer = renderer_set(self._renderer, NativeRenderer, self.model, self.model.P)
        return self._renderer.evaluate(cams, gts, self.bg, protocol=protocol, antialiasing=self.antialiasing, debug=self._debug.on)
