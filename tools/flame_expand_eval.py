"""Expansion kernel time for softmax weights (gs_flame shape: ~10k faces, K splats per face), per-thread kernels
(expand_wide = 0) against the warp-per-face kernels (expand_wide = 2), forward and backward, measured with the library's
CUDA-event spans.  Prints one JSON line per K; the expand_wide = 1 threshold (GMS_EXP_WIDE_MIN_K) comes from these.

    python tools/flame_expand_eval.py [--faces 9976] [--ks 1,3,7,16,32,64,100,128] [--reps 50]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")]

import torch  # noqa: E402

from gms_b200 import _lib, expansion  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--faces", type=int, default=9976)
    ap.add_argument("--ks", default="1,3,7,16,32,64,100,128")
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    import flame_driver
    rings = int(round((a.faces / 2) ** 0.5))
    drv = flame_driver.SyntheticFlame(rings=rings, segments=a.faces // (2 * rings))
    v = drv.v_template.cuda().contiguous()
    f = torch.from_numpy(drv.faces).cuda()
    F = f.shape[0]
    _lib.set_option("time_kernels", 1)
    for K in [int(k) for k in a.ks.split(",")]:
        al = torch.randn(F, K, 3, device="cuda", requires_grad=True)
        sc = torch.rand(F * K, 1, device="cuda", requires_grad=True)
        vv = v.clone().requires_grad_(True)
        row = dict(F=F, K=K)
        for wide in (0, 2):
            old = _lib.set_option("expand_wide", wide)
            for _ in range(3):
                xyz, s, r, _, _ = expansion.expand(vv, f, al, sc, alpha_activation=_lib.ALPHA_SOFTMAX)
                torch.autograd.backward((xyz, s, r), (torch.ones_like(xyz), torch.ones_like(s), torch.ones_like(r)))
            torch.cuda.synchronize()
            _lib.kernel_times(reset=True)
            for _ in range(a.reps):
                xyz, s, r, _, _ = expansion.expand(vv, f, al, sc, alpha_activation=_lib.ALPHA_SOFTMAX)
                torch.autograd.backward((xyz, s, r), (torch.ones_like(xyz), torch.ones_like(s), torch.ones_like(r)))
            torch.cuda.synchronize()
            t = _lib.kernel_times(reset=True)
            for k in ("expand_fwd", "expand_bwd"):
                row[f"{k}_ms_wide{wide}"] = round(t[k][0] / t[k][1], 5)
            _lib.set_option("expand_wide", old)
        row["gpu"] = torch.cuda.get_device_name()
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
