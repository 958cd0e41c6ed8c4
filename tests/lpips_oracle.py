"""A float64 restatement of VGG16 LPIPS v0.1 as lpipsPyTorch computes it (metrics.py:74 -> lpips(x, y, net_type='vgg')):

1. z-score per channel: (x - shift) / scale, shift = (-0.030, -0.088, -0.188), scale = (0.458, 0.448, 0.450); the input is
   NOT mapped from [0,1] to [-1,1] first (a quirk of lpipsPyTorch, reproduced).
2. torchvision vgg16().features up to relu5_3: LAYERS below, conv3x3 padding 1 with bias, ReLU, MaxPool2d(2, 2) (floor);
   the padding is zero in z-score space.
3. Target maps: the post-ReLU outputs at features' 1-based layers 4, 9, 16, 23, 30 (64, 128, 256, 512, 512 channels).
4. Each is normalised per pixel: f / (sqrt(sum_c f^2) + 1e-10).
5. Per layer: mean_{h,w} sum_c w_l[c] (fx - fy)^2, w_l the bias-free 1x1 lin conv.
6. LPIPS = the sum of the five terms.

Weights are the two state dicts (torchvision's vgg16 file, PerceptualSimilarity's vgg.pth)."""
import torch
import torch.nn.functional as F

SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
# torchvision vgg16().features[:30], written out: ("conv", index, Cin, Cout), ("relu",), ("pool",)
LAYERS = [
    ("conv", 0, 3, 64), ("relu",), ("conv", 2, 64, 64), ("relu",), ("pool",),
    ("conv", 5, 64, 128), ("relu",), ("conv", 7, 128, 128), ("relu",), ("pool",),
    ("conv", 10, 128, 256), ("relu",), ("conv", 12, 256, 256), ("relu",), ("conv", 14, 256, 256), ("relu",), ("pool",),
    ("conv", 17, 256, 512), ("relu",), ("conv", 19, 512, 512), ("relu",), ("conv", 21, 512, 512), ("relu",), ("pool",),
    ("conv", 24, 512, 512), ("relu",), ("conv", 26, 512, 512), ("relu",), ("conv", 28, 512, 512), ("relu",),
]
TARGET_LAYERS = (4, 9, 16, 23, 30)       # 1-based positions in LAYERS


def features(x: torch.Tensor, vgg16: dict, dtype=torch.float64) -> list:
    """The five target maps of x ([N,3,H,W]) in `dtype`."""
    dev = x.device
    x = x.to(dtype)
    shift = torch.tensor(SHIFT, dtype=torch.float32).to(dtype).to(dev).view(1, 3, 1, 1)
    scale = torch.tensor(SCALE, dtype=torch.float32).to(dtype).to(dev).view(1, 3, 1, 1)
    x = (x - shift) / scale
    out = []
    for i, layer in enumerate(LAYERS, 1):
        if layer[0] == "conv":
            idx = layer[1]
            x = F.conv2d(x, vgg16[f"features.{idx}.weight"].to(dev, dtype), vgg16[f"features.{idx}.bias"].to(dev, dtype), padding=1)
        elif layer[0] == "relu":
            x = F.relu(x)
        else:
            x = F.max_pool2d(x, 2, 2)
        if i in TARGET_LAYERS:
            out.append(x)
    return out


def normalize(f: torch.Tensor, eps: float = 1e-10) -> torch.Tensor:
    return f / (torch.sqrt(torch.sum(f ** 2, dim=1, keepdim=True)) + eps)


def head(fx: list, fy: list, lin: dict) -> torch.Tensor:
    """[6]: the five layer terms (steps 4-5) from the target maps of both images, then their sum."""
    terms = []
    for l, (a, b) in enumerate(zip(fx, fy)):
        w = lin[f"lin{l}.model.1.weight"].to(a.device, a.dtype)
        terms.append(F.conv2d((normalize(a) - normalize(b)) ** 2, w).mean((2, 3)).reshape(()))
    t = torch.stack(terms)
    return torch.cat([t, t.sum().reshape(1)])


def lpips(img: torch.Tensor, gt: torch.Tensor, vgg16: dict, lin: dict, dtype=torch.float64) -> torch.Tensor:
    """[6] in `dtype` for [3,H,W] img and gt; both run as one batch of two."""
    f = features(torch.stack([img, gt]), vgg16, dtype)
    return head([t[0:1] for t in f], [t[1:2] for t in f], lin)


LIN_CHANNELS = (64, 128, 256, 512, 512)


def seeded_state_dicts(seed: int = 0) -> tuple:
    """(vgg16 state dict, vgg.pth state dict) in the two files' real key formats: He-scaled conv weights, small biases,
    non-negative lin weights (as the published ones are), and a classifier entry the loader must ignore."""
    g = torch.Generator().manual_seed(seed)
    vgg16 = {}
    for layer in LAYERS:
        if layer[0] == "conv":
            _, idx, cin, cout = layer
            vgg16[f"features.{idx}.weight"] = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5
            vgg16[f"features.{idx}.bias"] = (torch.rand(cout, generator=g) - 0.5) * 0.1
    vgg16["classifier.0.weight"] = torch.randn(8, 16, generator=g)          # the real one is [4096, 25088]
    vgg16["classifier.0.bias"] = torch.randn(8, generator=g)
    lin = {f"lin{l}.model.1.weight": torch.rand(1, c, 1, 1, generator=g) * (2.0 / c) for l, c in enumerate(LIN_CHANNELS)}
    return vgg16, lin


def write_weight_files(directory, seed: int = 0) -> tuple:
    """Writes vgg16-397923af.pth and vgg.pth (torch.save, as torchvision and PerceptualSimilarity ship them) into
    `directory`; returns (vgg16 path, lin path, vgg16 state dict, lin state dict)."""
    import os
    vgg16, lin = seeded_state_dicts(seed)
    vp, lp = os.path.join(str(directory), "vgg16-397923af.pth"), os.path.join(str(directory), "vgg.pth")
    torch.save(vgg16, vp)
    torch.save(lin, lp)
    return vp, lp, vgg16, lin
