"""Debug mode of the native trainers: the reference's pipe.debug, `train.py --debug` and `--debug_from N`.

A debug step runs its one-call frame with settings.debug (every launch waited for and named on a fault, the binning check
on the frame's own buffers), and synchronises after every other library call the step makes, naming it.  Before the
frame, everything needed to repeat the step is copied to the host: the trainer's state_dict(), the model, the camera, the
background, the ground truth, the iteration, the active SH degree and the antialiasing setting.  The model is stored as its
structure: the parameters' values are in the state_dict() copy only.  When the step fails, the
copy is written with torch.save (the native counterpart of the rasterizer's snapshot_fw.dump), the reference's message is
printed and the error re-raised; replay(path) repeats that step.
"""
from __future__ import annotations

import copy
import ctypes
import io
from typing import Optional

import numpy as np
import torch

SNAPSHOT = "snapshot_frame.dump"


def to_host(obj):
    """Copies of every tensor in a (nested) dict / list / tuple on the host."""
    if torch.is_tensor(obj):
        return obj.detach().cpu().clone()
    if isinstance(obj, dict):
        return {k: to_host(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(to_host(v) for v in obj)
    return obj


def to_device(obj, dev):
    if torch.is_tensor(obj):
        return obj.to(dev)
    if isinstance(obj, dict):
        return {k: to_device(v, dev) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(to_device(v, dev) for v in obj)
    return obj


class _Slot:
    """Stands in, in a snapshot's model, for a tensor whose values the snapshot's state_dict() holds (a view of the
    optimizer's flat parameter buffer), or for a gradient buffer the model keeps: its shape, dtype and kind only."""

    def __init__(self, t: torch.Tensor):
        self.shape, self.dtype = tuple(t.shape), t.dtype
        self.param, self.requires_grad = isinstance(t, torch.nn.Parameter), bool(t.requires_grad)
        self.grad = t.grad is not None

    def make(self, dev) -> torch.Tensor:
        t = torch.zeros(self.shape, dtype=self.dtype, device=dev)
        t = torch.nn.Parameter(t, requires_grad=self.requires_grad) if self.param else t.requires_grad_(self.requires_grad)
        if self.grad:
            t.grad = torch.zeros_like(t)
        return t


def model_structure(model, flat: torch.Tensor):
    """A shallow copy of `model` to serialise: every tensor attribute that views the optimizer's flat buffer `flat` (its
    values are in the state_dict()) becomes a _Slot, and so does every tensor with a gradient buffer, which serialising
    would drop (a FlameGaussianModel's `vertices`, whose .grad the frame writes); ctypes caches (a segmented model's
    gms_mesh_segment array) are left out."""
    base = flat.untyped_storage().data_ptr()
    m = copy.copy(model)
    d = {}
    for k, v in model.__dict__.items():
        if isinstance(v, ctypes.Array):
            continue
        if torch.is_tensor(v) and (v.untyped_storage().data_ptr() == base or v.grad is not None):
            v = _Slot(v)
        d[k] = v
    m.__dict__ = d
    return m


def rebuild_model(m, dev):
    """The inverse of model_structure, on `dev`: _Slots become zero tensors of their shape (with a zero gradient buffer where
    the model kept one; the trainer's load_state_dict fills the parameters), and a segmented model gets its segment array."""
    for k, v in list(m.__dict__.items()):
        if isinstance(v, _Slot):
            setattr(m, k, v.make(dev))
    if getattr(m, "segments", None) is not None:
        from . import _lib
        m._segment_array = _lib.mesh_segments(m.segments)
    return m


def sync(what: str, dev) -> None:
    """A debug step's check after a library call queued outside the frame: wait for it and name it on a fault."""
    if torch.device(dev).type != "cuda":
        return
    try:
        torch.cuda.current_stream(dev).synchronize()
    except RuntimeError as e:
        raise RuntimeError(f"{what}: {e}") from e


class DebugMode:
    """The reference's rule for one trainer: debug=True from the first step; else on at the step whose iteration - 1 ==
    debug_from, and on from then on (a run resumed past debug_from never turns it on).  Not part of the trainer's state."""

    def __init__(self, debug: bool = False, debug_from: int = -1, snapshot: str = SNAPSHOT):
        self.on, self.debug_from, self.path = bool(debug), int(debug_from), str(snapshot)

    def begin(self, iteration: int) -> bool:
        """Whether step `iteration` (1-based) runs in debug mode."""
        if iteration - 1 == self.debug_from:
            self.on = True
        return self.on

    def snapshot(self, trainer, cam, gt: torch.Tensor, bg: torch.Tensor, iteration: int) -> dict:
        """The host copy of everything a replay of step `iteration` needs, taken before the frame runs."""
        model = io.BytesIO()
        torch.save(model_structure(trainer.model, trainer._debug_flat()), model)    # (copies its other device tensors to the host)
        return {"trainer": type(trainer).__name__, "config": trainer._debug_config(), "model": model.getvalue(),
                "state_dict": to_host(trainer.state_dict()),
                "camera": {"image_width": int(cam.image_width), "image_height": int(cam.image_height), "FoVx": float(cam.FoVx),
                           "FoVy": float(cam.FoVy), "world_view_transform": to_host(cam.world_view_transform),
                           "full_proj_transform": to_host(cam.full_proj_transform), "camera_center": to_host(cam.camera_center),
                           "uid": getattr(cam, "uid", None)},
                "bg": to_host(bg), "gt": to_host(gt), "iteration": int(iteration),
                "active_sh_degree": int(trainer.model.active_sh_degree), "antialiasing": bool(trainer.antialiasing)}

    def failed(self, snap: dict, err: BaseException) -> None:
        """Writes the snapshot and prints the reference's message (rasterizer's snapshot_fw.dump, adapted).  When the snapshot
        cannot be written, says so; the step's own error is still the one raised."""
        try:
            torch.save(snap, self.path)
        except Exception as e:
            print(f"\nAn error occured in the training frame: {err}. The snapshot could not be written to {self.path}: {e}")
            return
        print(f"\nAn error occured in the training frame: {err}. Please forward {self.path} for debugging.")


def run_step(trainer, step, cam, gt, bg, iteration: int):
    """A trainer's step `iteration` through step(debug): in debug mode the snapshot is taken first and, when the step
    raises, written, the trainer's state is put back from it (trainer._debug_restore; not after a device fault, which leaves
    nothing on the device to trust) and the error re-raised."""
    dbg = trainer._debug
    if not dbg.begin(iteration):
        return step(False)
    snap = dbg.snapshot(trainer, cam, gt, bg, iteration)
    try:
        return step(True)
    except Exception as e:
        dbg.failed(snap, e)
        try:
            trainer._debug_restore(snap)
        except Exception:       # a device fault: the snapshot is the record of the state
            pass
        raise


def frame_outputs(frame, cam) -> dict:
    """The image [3,H,W], radii [P] and inverse depth [1,H,W] a training frame left in its workspace for `cam`, and its loss
    vector, as copies."""
    import ctypes as C
    from . import _lib
    P = frame._gaussians()
    W, H = int(cam.image_width), int(cam.image_height)
    v = _lib.FrameView()
    _lib.check(_lib.lib().gms_frame_views(frame.ws.data_ptr(), P, W, H, C.byref(v)), "gms_frame_views")

    def take(ptr, shape, dtype=torch.float32):
        off = ptr - frame.ws.data_ptr()
        return frame.ws[off:off + 4 * int(np.prod(shape))].view(dtype).view(shape).clone()

    return dict(image=take(v.image, (3, H, W)), radii=take(v.radii, (P,), torch.int32), invdepth=take(v.invdepth, (1, H, W)),
                loss=frame.loss.clone())


def replay(path: str, device: Optional[torch.device] = None, snapshot: Optional[str] = None) -> dict:
    """Rebuilds a trainer of the snapshot's type from `path` (its model, state, iteration, SH degree) and runs the snapshot's
    step once with debug on.  Returns {"image", "radii", "invdepth", "loss"} of the step's frame, or raises the step's error
    (a failing replay writes its own snapshot to `snapshot`, default: the replayed file's name with ".replay")."""
    from .scenes import Camera
    from .trainer import FlameTrainer, FreeTrainer, MeshTrainer
    dev = torch.device(device or "cuda")
    snap = torch.load(path, map_location="cpu", weights_only=False)
    model = rebuild_model(torch.load(io.BytesIO(snap["model"]), map_location=dev, weights_only=False), dev)
    cls = {"MeshTrainer": MeshTrainer, "FreeTrainer": FreeTrainer, "FlameTrainer": FlameTrainer}[snap["trainer"]]
    bg = snap["bg"].to(dev)
    trainer = cls(model, bg, **snap["config"], debug=True, debug_snapshot=snapshot or f"{path}.replay")
    trainer._debug_restore(snap)
    c = snap["camera"]
    cam = Camera(c["image_width"], c["image_height"], c["FoVx"], c["FoVy"], c["world_view_transform"].to(dev),
                 c["full_proj_transform"].to(dev), c["camera_center"].to(dev), c["uid"])
    trainer.step(cam, snap["gt"].to(dev), bg=bg)
    out = frame_outputs(trainer.native_frame, cam)
    out["loss"] = out["loss"][0]
    return out
