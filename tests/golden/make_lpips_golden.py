"""Generate lpips.npz by running THE REFERENCE's own lpipsPyTorch/modules/lpips.py (LPIPS.forward) on given feature maps --
run in the build container only; the fixture is committed, the reference is never read at test time.

    python tests/golden/make_lpips_golden.py        (needs /root/reference)

lpips.py imports get_network / LinLayers from .networks and get_state_dict from .utils.  The reference's own networks.py
and utils.py are loaded (LinLayers and normalize_activation are theirs), with two stand-ins, so nothing is downloaded:
- networks.get_network returns a module whose forward(x) hands back normalize_activation of the given raw maps of the
  image that x names (x[0,0,0,0]: 0 the render, 1 the ground truth), as BaseNet.forward does with VGG16's target maps;
- utils.get_state_dict returns the given lin weights in vgg.pth's key format (lin{l}.model.1.weight), renamed as the
  reference renames them.
Stored per case: the raw target maps of both images (post-ReLU, [1,C,h,w], C = 64, 128, 256, 512, 512), the lin weights,
and the reference's output (float32 [1,1,1,1]).  Case 1 has a pixel whose maps are all zero in every layer (0 / (0 + 1e-10));
case 2 compares identical maps."""
import importlib.util
import os
import sys
import types
from collections import OrderedDict

import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
CHANNELS = (64, 128, 256, 512, 512)
SPATIAL = ((7, 5), (4, 3), (3, 2), (2, 2), (1, 2))


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def reference_lpips(maps_x, maps_y, lin):
    mods = os.path.join(REF, "lpipsPyTorch", "modules")
    for pkg in ("lp_ref", "lp_ref.modules"):
        m = types.ModuleType(pkg)
        m.__path__ = []
        sys.modules[pkg] = m
    utils = _load("lp_ref.modules.utils", os.path.join(mods, "utils.py"))
    networks = _load("lp_ref.modules.networks", os.path.join(mods, "networks.py"))

    class GivenMaps(torch.nn.Module):
        n_channels_list = list(CHANNELS)

        def forward(self, x):
            maps = maps_y if int(x[0, 0, 0, 0]) == 1 else maps_x
            return [utils.normalize_activation(f) for f in maps]

    def get_state_dict(net_type="vgg", version="0.1"):
        assert (net_type, version) == ("vgg", "0.1")
        return OrderedDict((k.replace("lin", "").replace("model.", ""), v) for k, v in lin.items())

    networks.get_network = lambda net_type: GivenMaps()
    utils.get_state_dict = get_state_dict
    lpips_mod = _load("lp_ref.modules.lpips", os.path.join(mods, "lpips.py"))
    crit = lpips_mod.LPIPS("vgg", "0.1")
    with torch.no_grad():
        return crit(torch.zeros(1, 3, 1, 1), torch.ones(1, 3, 1, 1))


def main():
    g = torch.Generator().manual_seed(3)
    out = {"n_cases": np.int64(3)}
    for case in range(3):
        lin = OrderedDict((f"lin{l}.model.1.weight", torch.rand(1, c, 1, 1, generator=g) * (2.0 / c)) for l, c in enumerate(CHANNELS))
        mx = [torch.relu(torch.randn(1, c, h, w, generator=g)) for c, (h, w) in zip(CHANNELS, SPATIAL)]
        my = [torch.relu(f + 0.5 * torch.randn(f.shape, generator=g)) for f in mx] if case != 2 else [f.clone() for f in mx]
        if case == 1:
            for f in mx + my:
                f[..., 0, 0] = 0.0
        res = reference_lpips(mx, my, lin)
        for l in range(5):
            out[f"case{case}_x{l}"] = mx[l].numpy()
            out[f"case{case}_y{l}"] = my[l].numpy()
            out[f"case{case}_lin{l}"] = lin[f"lin{l}.model.1.weight"].numpy()
        out[f"case{case}_lpips"] = res.numpy()
        print(f"case {case}: reference LPIPS {res.flatten().tolist()}")
    np.savez_compressed(os.path.join(HERE, "lpips.npz"), **out)


if __name__ == "__main__":
    main()
