"""LPIPS on the device: lpips(render, gt, net_type='vgg') as metrics.py:74 calls it (lpipsPyTorch, version 0.1), forward only.

    L = Lpips.from_cache()                        # the files a run of the reference's metrics.py leaves in the torch hub cache
    out = L.lpips(img, gt)                        # device float32 [6]: five layer terms, then LPIPS (LAYER_NAMES)

The weights are read from files already on disk and never fetched:
  <torch.hub.get_dir()>/checkpoints/vgg16-397923af.pth   torchvision's vgg16 ImageNet weights (features.* is used)
  <torch.hub.get_dir()>/checkpoints/vgg.pth              PerceptualSimilarity v0.1's lin layers (lin{0..4}.model.1.weight)
Both are read with torch.load(weights_only=True) and packed once, at load, into the layout gms_lpips_vgg reads
(include/gms_b200.h).  DESIGN.md 4.8 restates the definition and the kernels."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

from . import _lib

VGG16_FILE = "vgg16-397923af.pth"
LIN_FILE = "vgg.pth"
LAYER_NAMES = ("relu1_2", "relu2_2", "relu3_3", "relu4_3", "relu5_3", "lpips")
# torchvision vgg16().features: the indices of the 13 convs and their (Cin, Cout); lin widths of the five target maps
CONV_INDEX = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
CONV_CHANNELS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512),
                 (512, 512), (512, 512), (512, 512), (512, 512))
LIN_CHANNELS = (64, 128, 256, 512, 512)
MIN_SIDE = 16


def cache_dir() -> str:
    """<torch.hub.get_dir()>/checkpoints, where torchvision and load_state_dict_from_url keep downloaded weights."""
    return os.path.join(torch.hub.get_dir(), "checkpoints")


def _load(path: str, what: str, other: str) -> dict:
    if not os.path.isfile(path):
        raise FileNotFoundError(f"LPIPS weights not found: {what} {path!r} is missing (expected with {other!r}). "
                                f"This library does not download weights; run the reference's metrics.py once, or copy "
                                f"the two files there.")
    return torch.load(path, map_location="cpu", weights_only=True)


def _tensor(sd: dict, key: str, shape: tuple, path: str) -> torch.Tensor:
    if key not in sd:
        raise KeyError(f"LPIPS weights: {path!r} has no key {key!r}")
    t = sd[key]
    if not isinstance(t, torch.Tensor) or tuple(t.shape) != shape:
        got = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
        raise ValueError(f"LPIPS weights: {path!r} key {key!r} has shape {got}, expected {shape}")
    return t.detach().to(torch.float32)


def pack_weights(vgg16: dict, lin: dict, vgg16_path: str = "vgg16", lin_path: str = "lin") -> torch.Tensor:
    """The float32 CPU vector gms_lpips_vgg reads (include/gms_b200.h), from the two state dicts.  Only features.<conv>.weight
    / .bias and lin{l}.model.1.weight are read; every other key (classifier.*) is ignored."""
    parts = []
    for i, (idx, (cin, cout)) in enumerate(zip(CONV_INDEX, CONV_CHANNELS)):
        w = _tensor(vgg16, f"features.{idx}.weight", (cout, cin, 3, 3), vgg16_path)
        b = _tensor(vgg16, f"features.{idx}.bias", (cout,), vgg16_path)
        w = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin)             # K ordered (ky, kx, ci)
        if i == 0:
            w = torch.cat([w, w.new_zeros(cout, 32 - 27)], 1)        # conv1_1: K padded to 32
        parts += [w.reshape(-1), b]
    for l, c in enumerate(LIN_CHANNELS):
        parts.append(_tensor(lin, f"lin{l}.model.1.weight", (1, c, 1, 1), lin_path).reshape(-1))
    packed = torch.cat(parts).contiguous()
    assert packed.numel() == _lib.LPIPS_WEIGHT_FLOATS
    return packed


def scratch_bytes(height: int, width: int) -> int:
    return int(_lib.lib().gms_lpips_scratch_bytes(int(height), int(width)))


class Lpips:
    """VGG16 LPIPS with its weights packed on one device.  lpips() enqueues on the current stream and never synchronises."""

    def __init__(self, packed: torch.Tensor, device="cuda"):
        if packed.dtype != torch.float32 or packed.numel() != _lib.LPIPS_WEIGHT_FLOATS:
            raise ValueError(f"Lpips: packed weights must be float32 [{_lib.LPIPS_WEIGHT_FLOATS}]")
        self.dev = torch.device(device)
        if self.dev.type != "cuda":
            raise RuntimeError("Lpips: a CUDA device is required (no CPU path in the product)")
        if self.dev.index is None:
            self.dev = torch.device("cuda", torch.cuda.current_device())
        self.weights = packed.to(self.dev).contiguous()
        self._scratch = None

    @classmethod
    def from_files(cls, vgg16_path: str, lin_path: str, device="cuda") -> "Lpips":
        """From torchvision's vgg16 state dict file and PerceptualSimilarity's vgg.pth."""
        vgg16 = _load(vgg16_path, "the VGG16 weights", lin_path)
        lin = _load(lin_path, "the LPIPS lin weights", vgg16_path)
        return cls(pack_weights(vgg16, lin, vgg16_path, lin_path), device)

    @classmethod
    def from_cache(cls, dir: Optional[str] = None, device="cuda") -> "Lpips":
        """From `dir` (default: cache_dir()), holding vgg16-397923af.pth and vgg.pth."""
        d = cache_dir() if dir is None else dir
        return cls.from_files(os.path.join(d, VGG16_FILE), os.path.join(d, LIN_FILE), device)

    def lpips(self, img: torch.Tensor, gt: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """LPIPS of float32 [3,H,W] `img` against `gt` (values as the reference's to_tensor gives them, [0,1]; not
        rescaled).  Returns `out` (device float32 [6], LAYER_NAMES), written in stream order."""
        if img.dim() != 3 or img.shape[0] != 3 or img.shape != gt.shape:
            raise ValueError(f"lpips: img and gt must both be [3,H,W]; got {tuple(img.shape)} and {tuple(gt.shape)}")
        for t, what in ((img, "img"), (gt, "gt")):
            if not t.is_cuda or t.device != self.dev or t.dtype != torch.float32:
                raise RuntimeError(f"lpips: {what} must be a float32 CUDA tensor on {self.dev}")
        _, H, W = img.shape
        if H < MIN_SIDE or W < MIN_SIDE:
            raise ValueError(f"lpips: images must be at least {MIN_SIDE}x{MIN_SIDE} (VGG16's fourth pooling); got {W}x{H}")
        img, gt = img.detach().contiguous(), gt.detach().contiguous()
        need = scratch_bytes(H, W)
        if self._scratch is None or self._scratch.numel() < need:
            self._scratch = None
            self._scratch = torch.empty(need, dtype=torch.uint8, device=self.dev)
        if out is None:
            out = torch.empty(6, dtype=torch.float32, device=self.dev)
        if out.dtype != torch.float32 or out.numel() != 6 or not out.is_contiguous() or out.device != self.dev:
            raise RuntimeError("lpips: out must be a contiguous float32 [6] tensor on the weights' device")
        a = _lib.LpipsArgs()
        a.H, a.W, a.img, a.gt, a.weights = H, W, img.data_ptr(), gt.data_ptr(), self.weights.data_ptr()
        a.out, a.scratch, a.scratch_bytes = out.data_ptr(), self._scratch.data_ptr(), self._scratch.numel()
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().gms_lpips_vgg(C.byref(a), torch.cuda.current_stream(self.dev).cuda_stream), "gms_lpips_vgg")
        return out
