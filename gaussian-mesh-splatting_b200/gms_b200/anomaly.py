"""Anomaly detection for native training: the reference's `train.py --detect_anomaly`.

The reference calls torch.autograd.set_detect_anomaly(True): the first backward function that returns NaN raises, names
itself, and the iteration stops before optimizer.step().  The one-call frames (gms_train_frame, gms_free_train_frame) run
their backward passes without an autograd graph, so here each backward stage's outputs are scanned for NaN on the device
right after the stage (gms_nan_scan), into one 64-bit record: key = stage << 56 | tensor << 48 | flat index, the smallest
key seen, so the record names the earliest stage, then the lowest tensor id, then the lowest row-major index.  A trainer
reads the record once per step and raises AnomalyError, with the location decoded, before any parameter changes.
"""
from __future__ import annotations

import bisect
import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib

# every stage a training frame has (each frame ignores the bit of the one it does not have: expansion or activation)
FRAME_STAGES = sum(1 << s for s in (_lib.ANOMALY_LOSS, _lib.ANOMALY_COMPOSITE_BWD, _lib.ANOMALY_PREPROCESS_BWD,
                                    _lib.ANOMALY_EXPAND_BWD, _lib.ANOMALY_ACTIVATION_BWD))

STAGE_NAMES = ("loss", "composite backward", "preprocess backward", "expansion backward", "activation backward", "FLAME backward")
TENSOR_NAMES = (("dL/dimage",),
                ("per-Gaussian gradient records",),
                ("dL/dmeans3D", "dL/dscales", "dL/drotations", "dL/dopacity_raw", "dL/dSH", "dL/dcolor_sh"),
                ("d_vertices", "d_alpha_raw", "d_scale_raw"),
                ("d_scaling_raw", "d_rotation_raw", "accum"),
                ("d_shape", "d_expression", "d_pose", "d_neck_pose", "d_transl", "d_enlargement"))

_INDEX_BITS = 48


def encode(stage: int, tensor: int, index: int) -> int:
    """The record key of a NaN at flat `index` of `tensor` in `stage`."""
    if not (0 <= stage < _lib.ANOMALY_STAGES and 0 <= tensor < 256 and 0 <= index < 1 << _INDEX_BITS):
        raise ValueError(f"anomaly key out of range: stage {stage}, tensor {tensor}, index {index}")
    return stage << 56 | tensor << 48 | index


def decode(key: int) -> Optional[Tuple[int, int, int]]:
    """(stage, tensor, index) of a record, or None for ANOMALY_NONE (no NaN found)."""
    key = int(key) & _lib.ANOMALY_NONE
    if key == _lib.ANOMALY_NONE:
        return None
    return key >> 56, (key >> 48) & 0xFF, key & ((1 << _INDEX_BITS) - 1)


@dataclass
class Layout:
    """What decoding a record needs to know about the frame: the view's size, the SH rows per Gaussian, the scale columns of
    free Gaussians, and for mesh-based models the (F_i, K_i) of each mesh (segments) -- `meshes` says whether a Gaussian is
    reported as (mesh, face, splat) (gs_mesh, gs_multi_mesh) or as (face, splat) (gs_flame, one mesh)."""
    H: int
    W: int
    M: int = 16
    scale_cols: int = 3
    segments: Optional[List[Tuple[int, int]]] = None
    meshes: bool = True


def layout_of(model, cam) -> Layout:
    """The Layout of a training frame of `model` drawing `cam`."""
    from .model import FlameGaussianModel, FreeGaussianModel
    H, W, M = int(cam.image_height), int(cam.image_width), int(model._features.shape[1])
    if isinstance(model, FreeGaussianModel):
        return Layout(H, W, M, scale_cols=int(model.scale_cols))
    F, K, _ = model.frame_sizes()
    segs = list(model.segments) if model.segments is not None else [(int(F), int(K))]
    return Layout(H, W, M, segments=segs, meshes=not isinstance(model, FlameGaussianModel))


def gaussian_of(row: int, segments: Sequence[Tuple[int, int]]) -> Tuple[int, int, int]:
    """(mesh, face within the mesh, splat) of Gaussian `row`: mesh i holds the rows [P_i, P_i + F_i K_i), face-major."""
    starts, p = [], 0
    for F, K in segments:
        starts.append(p)
        p += F * K
    if not 0 <= row < p:
        raise ValueError(f"Gaussian {row} outside the model's {p}")
    i = bisect.bisect_right(starts, row) - 1
    face, splat = divmod(row - starts[i], segments[i][1])
    return i, face, splat


def _row_width(stage: int, tensor: int, lay: Layout) -> int:
    """Floats per Gaussian of a per-Gaussian tensor."""
    if stage == _lib.ANOMALY_COMPOSITE_BWD:
        return 12
    if stage == _lib.ANOMALY_PREPROCESS_BWD:
        return (3, 3, 4, 1, 3 * lay.M, 3)[tensor]
    if stage == _lib.ANOMALY_EXPAND_BWD:
        return (3, 3, 1)[tensor]
    return (lay.scale_cols, 4, 1)[tensor]       # activation backward


def locate(stage: int, tensor: int, index: int, lay: Layout) -> str:
    """Where flat `index` of the tensor lies: (channel, y, x) of dL/dimage, (vertex, coordinate) of a vertex gradient, the
    element of a FLAME parameter, else the Gaussian row and column, with its (mesh, face, splat) for mesh-based models."""
    if stage == _lib.ANOMALY_LOSS:
        c, r = divmod(index, lay.H * lay.W)
        y, x = divmod(r, lay.W)
        return f"channel {c}, y {y}, x {x}"
    if (stage, tensor) in ((_lib.ANOMALY_EXPAND_BWD, _lib.ANOMALY_DVERTICES), (_lib.ANOMALY_FLAME_BWD, _lib.ANOMALY_DENLARGEMENT)):
        v, c = divmod(index, 3)
        return f"vertex {v}, coordinate {c}"
    if stage == _lib.ANOMALY_FLAME_BWD:
        return f"element {index}"
    row, col = divmod(index, _row_width(stage, tensor, lay))
    where = f"Gaussian {row}, column {col}"
    if lay.segments:
        mesh, face, splat = gaussian_of(row, lay.segments)
        where += f" (mesh {mesh}, face {face}, splat {splat})" if lay.meshes else f" (face {face}, splat {splat})"
    return where


class AnomalyError(RuntimeError):
    """A backward stage of a native training frame returned NaN (train.py --detect_anomaly).  Raised by a trainer's step()
    before any parameter, optimizer moment, step count or statistic changed.  stage / tensor / index: the record's fields;
    stage_name / tensor_name / location: their meaning."""

    def __init__(self, key: int, lay: Layout, iteration: Optional[int] = None):
        self.key = int(key) & _lib.ANOMALY_NONE
        self.stage, self.tensor, self.index = decode(self.key)
        self.stage_name = STAGE_NAMES[self.stage]
        names = TENSOR_NAMES[self.stage]
        self.tensor_name = names[self.tensor] if self.tensor < len(names) else f"tensor {self.tensor}"
        self.location = locate(self.stage, self.tensor, self.index, lay)
        at = "" if iteration is None else f" at iteration {iteration}"
        super().__init__(f"Function '{self.stage_name}' returned nan values in its output {self.tensor_name} (stage "
                         f"{self.stage}, tensor {self.tensor}){at}: first at flat index {self.index}, {self.location}")


def nan_scan(record: torch.Tensor, stage: int, buffers: Sequence[Tuple[int, torch.Tensor]]) -> None:
    """gms_nan_scan of `buffers` ((tensor id, float32 CUDA tensor), at most NAN_SCAN_MAX_BUFFERS) into `record` (int64 [1]
    on the device, the uint64 word) on the current stream."""
    a = _lib.NanScanArgs()
    if len(buffers) > _lib.NAN_SCAN_MAX_BUFFERS:
        raise ValueError(f"nan_scan: at most {_lib.NAN_SCAN_MAX_BUFFERS} buffers per call")
    for i, (tid, t) in enumerate(buffers):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.device != record.device:
            raise ValueError(f"nan_scan: buffer {i} must be a contiguous float32 tensor on {record.device}")
        a.buffers[i].ptr, a.buffers[i].n, a.buffers[i].tensor = t.data_ptr(), t.numel(), int(tid)
    a.n_buffers, a.stage, a.record = len(buffers), int(stage), record.data_ptr()
    with torch.cuda.device(record.device):
        _lib.check(_lib.lib().gms_nan_scan(C.byref(a), torch.cuda.current_stream(record.device).cuda_stream), "gms_nan_scan")


class AnomalyRecord:
    """The device record of one trainer: reset() before a frame, the frame's hooks (and scan()) write it, read() takes it to the
    host with one synchronisation."""

    def __init__(self, dev):
        self.word = torch.full((1,), -1, dtype=torch.int64, device=dev)     # all ones: ANOMALY_NONE

    @property
    def ptr(self) -> int:
        return self.word.data_ptr()

    def reset(self) -> "AnomalyRecord":
        self.word.fill_(-1)
        return self

    def scan(self, stage: int, buffers: Sequence[Tuple[int, torch.Tensor]]) -> None:
        nan_scan(self.word, stage, buffers)

    def read(self) -> int:
        return int(self.word.item()) & _lib.ANOMALY_NONE

    def check(self, lay: Layout, iteration: Optional[int] = None) -> None:
        """Raise AnomalyError if the record holds a NaN's key."""
        key = self.read()
        if key != _lib.ANOMALY_NONE:
            raise AnomalyError(key, lay, iteration)
