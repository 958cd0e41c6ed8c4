"""A whole gs_flame training step, native against the reference's op sequence.

    python tools/flame_train_eval.py --bench [--faces 9976] [--K 100] [--width 1920 --height 1080] [--steps 30] [--rounds 3]

Arms, alternated round by round on the same model start and 16 ring cameras (random ground truth):
  native   FlameTrainer: the driver in ATen, one gms_train_frame with softmax weights, autograd through the driver, FlatAdam;
  autograd tests/flame_reference.AtenFlameArm: ATen softmax expansion, shim rasterizer, fused loss, torch.optim.Adam (11 groups).
The driver is tests/flame_driver.SyntheticFlame (FLAME-shaped LBS).  Prints one JSON line: ms/step of both arms (median over
rounds), library launches per native step, the driver's share of the native step (its forward + backward alone, timed
with CUDA events), and the expand_fwd / expand_bwd spans inside the native step."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gms_b200 import _lib, scenes  # noqa: E402
from gms_b200.model import FlameGaussianModel  # noqa: E402
from gms_b200.trainer import FlameTrainer  # noqa: E402


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for i in range(n):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--faces", type=int, default=9976)
    ap.add_argument("--K", type=int, default=100)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import flame_driver
    import flame_reference as fr
    rings = int(round((a.faces / 2) ** 0.5))
    drv = flame_driver.SyntheticFlame(rings=rings, segments=a.faces // (2 * rings)).cuda()
    faces = torch.from_numpy(drv.faces).cuda()
    W, H = a.width, a.height
    cams = [scenes.look_at_camera((0.35 * np.cos(t), 0.1, 0.35 * np.sin(t)), (0, 0, 0), W, H).to("cuda")
            for t in np.linspace(0, 2 * np.pi, 16, endpoint=False)]
    g = torch.Generator(device="cuda").manual_seed(0)
    gts = [torch.rand(3, H, W, device="cuda", generator=g) for _ in cams]
    bg = torch.ones(3, device="cuda")
    m = FlameGaussianModel.create(drv, faces, K=a.K, seed=0)
    m.active_sh_degree = 3
    arm = fr.AtenFlameArm(m, bg)
    t = FlameTrainer(m, bg)
    nat, aut = [], []
    for _ in range(a.rounds):
        timed(lambda i: t.step(cams[i % 16], gts[i % 16]), 3)
        nat.append(timed(lambda i: t.step(cams[i % 16], gts[i % 16]), a.steps))
        timed(lambda i: arm.step(cams[i % 16], gts[i % 16]), 3)
        aut.append(timed(lambda i: arm.step(cams[i % 16], gts[i % 16]), a.steps))
    _lib.launch_count(reset=True)
    timed(lambda i: t.step(cams[i % 16], gts[i % 16]), 10)
    launches = _lib.launch_count() / 10

    def driver(i):
        v = m.driver_vertices()
        torch.autograd.backward(v, m.vertices.grad)
    drv_ms = timed(driver, a.steps)
    t.adam.zero_grad()
    spans = {}
    _lib.set_option("time_kernels", 1)
    timed(lambda i: t.step(cams[i % 16], gts[i % 16]), 3)
    _lib.kernel_times(reset=True)
    timed(lambda i: t.step(cams[i % 16], gts[i % 16]), a.steps)
    kt = _lib.kernel_times(reset=True)
    for k in ("expand_fwd", "expand_bwd"):
        spans[f"{k}_ms"] = round(kt[k][0] / kt[k][1], 4)
    _lib.set_option("time_kernels", 0)
    nm = statistics.median(nat)
    print(json.dumps(dict(F=m.faces.shape[0], K=a.K, P=m.P, width=W, height=H, cameras=16, native_ms_per_step=round(nm, 3),
                          native_ms_rounds=[round(x, 3) for x in nat], autograd_ms_per_step=round(statistics.median(aut), 3),
                          autograd_ms_rounds=[round(x, 3) for x in aut], library_launches_per_native_step=launches,
                          driver_fwd_bwd_ms=round(drv_ms, 3), driver_share_of_native_step=round(drv_ms / nm, 3), **spans,
                          gpu=torch.cuda.get_device_name())), flush=True)


if __name__ == "__main__":
    main()
