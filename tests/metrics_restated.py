"""Float64 restatement of the four view metrics of gms_image_metrics (gms_b200.metrics.METRIC_NAMES), written from their
definitions: L1 = mean |x - y| (utils/loss_utils.py:17); SSIM with an 11x11 Gaussian window, sigma 1.5, zero padding,
mean (utils/loss_utils.py:33-64); PSNR = -10 log10(MSE) over all channels, and the mean of the per-channel PSNRs
(utils/image_utils.py:17-19 on a [1,C,H,W] and on a [C,H,W] tensor).  Both images first go through the protocol's
transform, evaluated in float32 exactly as the reference evaluates it."""
import math

import torch


def transform(x: torch.Tensor, protocol: str) -> torch.Tensor:
    x = x.detach().cpu().float()
    if protocol == "training_report":
        return x.clamp(0.0, 1.0)                                                # train.py:203-204
    if protocol == "metrics":
        b = x.mul(255).add(0.5).clamp(0, 255).to(torch.uint8)                  # torchvision save_image
        return b.float().div(255)                                               # ToTensor on the saved PNG
    raise ValueError(protocol)


def metrics64(img: torch.Tensor, gt: torch.Tensor, protocol: str) -> list:
    x, y = transform(img, protocol).double(), transform(gt, protocol).double()
    Cn = x.shape[0]
    g = torch.tensor([math.exp(-(k - 5) ** 2 / (2 * 1.5 ** 2)) for k in range(11)], dtype=torch.float64)
    g = g / g.sum()
    win = (g[:, None] * g[None, :]).expand(Cn, 1, 11, 11).contiguous()
    conv = lambda t: torch.nn.functional.conv2d(t[None], win, padding=5, groups=Cn)[0]
    mu1, mu2 = conv(x), conv(y)
    s1, s2, s12 = conv(x * x) - mu1 * mu1, conv(y * y) - mu2 * mu2, conv(x * y) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim = ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s1 + s2 + C2))
    d = x - y
    psnr = lambda mse: -10.0 * math.log10(mse) if mse > 0 else math.inf
    mse_c = (d * d).reshape(Cn, -1).mean(1)
    return [float(d.abs().mean()), float(ssim.mean()), psnr(float((d * d).mean())),
            sum(psnr(float(m)) for m in mse_c) / Cn]
