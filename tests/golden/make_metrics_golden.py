"""Generate metrics.npz by IMPORTING THE REFERENCE's own metric functions (/root/reference) -- run in the build container
only; the fixture is committed, the reference is never read at test time.

    python tests/golden/make_metrics_golden.py

For seeded image pairs (values a little outside [0, 1], so that the clamp and the 8-bit rounding matter), both protocols:
  training_report  clamp (train.py:203-204), l1_loss / ssim (utils/loss_utils.py:17, :33-64), psnr on the [C,H,W] tensors
                   (utils/image_utils.py:17-19; one PSNR per channel, train.py:212 averages them) and on [1,C,H,W]
  metrics          save_image's rounding and ToTensor's byte / 255 (scripts/render.py -> metrics.py:36-45), then ssim and psnr
                   on [1,C,H,W] (metrics.py:72-73)
Each case stores img, gt and, per protocol, [L1, SSIM, PSNR over all channels, mean of the per-channel PSNRs]."""
import os
import sys

import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)

from utils.image_utils import psnr as ref_psnr  # noqa: E402
from utils.loss_utils import l1_loss as ref_l1, ssim as ref_ssim  # noqa: E402

CASES = [(3, 45, 70, 0.15), (3, 40, 33, 0.05), (3, 37, 52, 0.3), (3, 32, 32, 0.0)]     # (C, H, W, noise); noise 0: identical images


def save_load_roundtrip(x):
    """torchvision.utils.save_image's byte (grid.mul(255).add_(0.5).clamp_(0, 255) ... to(uint8)), then ToTensor (byte / 255)."""
    return x.mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8).float().div(255)


def scores(a, b, protocol):
    if protocol == "training_report":
        a, b = torch.clamp(a, 0.0, 1.0), torch.clamp(b, 0.0, 1.0)
    else:
        a, b = save_load_roundtrip(a.clone()), save_load_roundtrip(b.clone())
    return np.array([ref_l1(a, b).item(), ref_ssim(a[None], b[None]).item(), ref_psnr(a[None], b[None]).mean().item(),
                     ref_psnr(a, b).mean().item()], np.float64)


def main():
    out = {}
    for i, (Cn, H, W, noise) in enumerate(CASES):
        g = torch.Generator().manual_seed(100 + i)
        img = torch.rand(Cn, H, W, generator=g) * 1.2 - 0.1
        gt = img + noise * torch.randn(Cn, H, W, generator=g) if noise else img.clone()
        out[f"case{i}_img"], out[f"case{i}_gt"] = img.numpy(), gt.numpy()
        for protocol in ("training_report", "metrics"):
            out[f"case{i}_{protocol}"] = scores(img, gt, protocol)
    out["n_cases"] = np.int64(len(CASES))
    np.savez_compressed(os.path.join(HERE, "metrics.npz"), **out)


if __name__ == "__main__":
    main()
    print("metrics.npz", os.path.getsize(os.path.join(HERE, "metrics.npz")))
