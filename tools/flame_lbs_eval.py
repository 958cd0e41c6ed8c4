"""FLAME's vertex model, native against ATen, and the gs_flame training step with each driver.

    python tools/flame_lbs_eval.py --bench [--faces 9940] [--K 100] [--width 1920 --height 1080] [--steps 30] [--rounds 3]

Arms, alternated round by round:
  lbs      gms_flame_lbs_forward + gms_flame_lbs_backward alone (six launches), against tests/flame_driver.SyntheticFlame's
           ATen forward + backward on the same buffers (FLAME's 100 shape + 50 expression columns, 36 pose features);
  step     a whole FlameTrainer step (tools/flame_train_eval.py's workload) with a NativeFlame driver and with the ATen driver.
The basis the kernels read is counted, not timed: (n_shape + n_exp) x 3V floats of shapedirs plus 36 x 3V of posedirs, per
direction.  Prints one JSON line with the card's name and power limit and library launches per step."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gms_b200 import _lib, scenes  # noqa: E402
from gms_b200.flame import NativeFlame  # noqa: E402
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


def power_limit():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--faces", type=int, default=9940)
    ap.add_argument("--K", type=int, default=100)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("flame_lbs_eval: needs a GPU")
    import flame_driver
    rings = int(round((a.faces / 2) ** 0.5))
    syn = flame_driver.SyntheticFlame(rings=rings, segments=a.faces // (2 * rings)).cuda()
    buf = dict(v_template=syn.v_template, shapedirs=syn.shapedirs, posedirs=syn.posedirs, J_regressor=syn.J_regressor,
               parents=flame_driver.PARENTS, lbs_weights=syn.lbs_weights, faces=syn.faces)
    nat = NativeFlame(**buf)
    V, B = nat.V, nat.n_shape + nat.n_exp
    faces = torch.from_numpy(syn.faces).cuda()
    W, H = a.width, a.height
    cams = [scenes.look_at_camera((0.35 * np.cos(t), 0.1, 0.35 * np.sin(t)), (0, 0, 0), W, H).to("cuda")
            for t in np.linspace(0, 2 * np.pi, 16, endpoint=False)]
    g = torch.Generator(device="cuda").manual_seed(0)
    gts = [torch.rand(3, H, W, device="cuda", generator=g) for _ in cams]
    bg = torch.ones(3, device="cuda")
    m_n = FlameGaussianModel.create(nat, faces, K=a.K, seed=0)
    m_a = FlameGaussianModel.create(syn, faces, K=a.K, seed=0)
    for m in (m_n, m_a):
        m.active_sh_degree = 3
    t_n, t_a = FlameTrainer(m_n, bg), FlameTrainer(m_a, bg)

    # the LBS alone, on model m_n's parameters and a fixed vertex gradient
    t_n.step(cams[0], gts[0])
    lbs = nat.bind(m_n)
    up = m_n.vertices.grad.clone()

    def native_lbs(i):
        lbs.forward()
        m_n.vertices.grad.copy_(up)
        lbs.backward()

    def aten_lbs(i):
        v = m_a.driver_vertices()
        torch.autograd.backward(v, up)

    copy_ms = timed(lambda i: m_n.vertices.grad.copy_(up), a.steps)
    lbs_n, lbs_a, step_n, step_a = [], [], [], []
    for _ in range(a.rounds):
        timed(native_lbs, 3)
        lbs_n.append(timed(native_lbs, a.steps) - copy_ms)
        timed(aten_lbs, 3)
        lbs_a.append(timed(aten_lbs, a.steps))
        timed(lambda i: t_n.step(cams[i % 16], gts[i % 16]), 3)
        step_n.append(timed(lambda i: t_n.step(cams[i % 16], gts[i % 16]), a.steps))
        timed(lambda i: t_a.step(cams[i % 16], gts[i % 16]), 3)
        step_a.append(timed(lambda i: t_a.step(cams[i % 16], gts[i % 16]), a.steps))
    t_a.adam.zero_grad()
    launches = {}
    for name, t in (("native", t_n), ("aten", t_a)):
        _lib.launch_count(reset=True)
        timed(lambda i: t.step(cams[i % 16], gts[i % 16]), 10)
        launches[name] = _lib.launch_count() / 10
    med = lambda xs: round(statistics.median(xs), 4)
    basis_mb = (B + 36) * 3 * V * 4 / 1e6
    print(json.dumps(dict(V=V, F=int(faces.shape[0]), K=a.K, P=m_n.P, width=W, height=H, n_shape=nat.n_shape, n_exp=nat.n_exp,
                          basis_mb_per_direction=round(basis_mb, 2),
                          lbs_native_fwd_bwd_ms=med(lbs_n), lbs_native_rounds=[round(x, 4) for x in lbs_n],
                          lbs_aten_fwd_bwd_ms=med(lbs_a), lbs_aten_rounds=[round(x, 4) for x in lbs_a],
                          step_native_lbs_ms=med(step_n), step_native_lbs_rounds=[round(x, 3) for x in step_n],
                          step_aten_driver_ms=med(step_a), step_aten_driver_rounds=[round(x, 3) for x in step_a],
                          library_launches_per_step_native_lbs=launches["native"], library_launches_per_step_aten_driver=launches["aten"],
                          gpu=torch.cuda.get_device_name(), power_limit=power_limit())), flush=True)


if __name__ == "__main__":
    main()
