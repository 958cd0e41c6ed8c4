"""Image quality of a rendered view against its ground truth on the device: L1, SSIM and two PSNRs (gms_image_metrics).

Two protocols of the reference, which differ only in what both images go through first:
  "training_report"  clamp to [0, 1]: train.py:203-204 (training_report on the test cameras)
  "metrics"          save_image's 8-bit rounding and back to byte / 255: scripts/render.py writes PNGs, metrics.py reads them
Row layout of the result (float64): METRIC_NAMES.  "psnr" is utils/image_utils.py:psnr over all channels of a [1,C,H,W]
batch (metrics.py:73); "psnr_per_channel" is the mean of the same psnr applied to a [C,H,W] tensor, whose view(shape[0], -1)
makes one PSNR per channel -- what training_report averages (train.py:212).  A PSNR is +inf where the MSE is 0."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib

PROTOCOLS = {"training_report": 0, "metrics": 1}
METRIC_NAMES = ("l1", "ssim", "psnr", "psnr_per_channel")


def scratch_bytes(channels: int, height: int, width: int) -> int:
    n = C.c_size_t(0)
    _lib.check(_lib.lib().gms_metrics_scratch_bytes(int(channels), int(height), int(width), C.byref(n)), "gms_metrics_scratch_bytes")
    return int(n.value)


def image_metrics(img: torch.Tensor, gt: torch.Tensor, protocol: str = "training_report", out: Optional[torch.Tensor] = None,
                  scratch: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Scores float [C,H,W] `img` against `gt` on the current stream.  Returns `out` (device float64 [4], METRIC_NAMES),
    written in stream order: nothing synchronises.  `scratch` (uint8, scratch_bytes()) may be reused across calls."""
    if protocol not in PROTOCOLS:
        raise ValueError(f"image_metrics: protocol must be one of {sorted(PROTOCOLS)}, got {protocol!r}")
    if img.dim() != 3 or img.shape != gt.shape:
        raise ValueError(f"image_metrics: img and gt must both be [C,H,W]; got {tuple(img.shape)} and {tuple(gt.shape)}")
    dev = img.device
    for t, what in ((img, "img"), (gt, "gt")):
        if not t.is_cuda or t.device != dev or t.dtype != torch.float32:
            raise RuntimeError(f"image_metrics: {what} must be a float32 CUDA tensor on {dev}")
    img, gt = img.detach().contiguous(), gt.detach().contiguous()
    Cn, H, W = img.shape
    need = scratch_bytes(Cn, H, W)
    if scratch is None or scratch.numel() < need:
        scratch = torch.empty(need, dtype=torch.uint8, device=dev)
    if out is None:
        out = torch.empty(4, dtype=torch.float64, device=dev)
    if out.dtype != torch.float64 or out.numel() != 4 or not out.is_contiguous() or out.device != dev:
        raise RuntimeError("image_metrics: out must be a contiguous float64 [4] tensor on the images' device")
    a = _lib.MetricsArgs()
    a.C, a.H, a.W, a.img, a.gt = Cn, H, W, img.data_ptr(), gt.data_ptr()
    a.quantize, a.out, a.scratch, a.scratch_bytes = PROTOCOLS[protocol], out.data_ptr(), scratch.data_ptr(), scratch.numel()
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().gms_image_metrics(C.byref(a), torch.cuda.current_stream(dev).cuda_stream), "gms_image_metrics")
    return out
