"""Training with antialiasing: what the reference's pipe.antialiasing costs a native training step.

    python tools/train_antialiasing_eval.py --bench [--parent DIR] [--out FILE]

Workloads:
  gs_mesh  MeshTrainer (native, Adam on): scenes.object_mesh(--faces) at K = 5 (1M mesh-Gaussians at the default 200k faces),
           1920x1080, --views ring cameras, seeded uint8 noise as ground truth.
  gs_flat  FreeTrainer (no densification in the window): 1M scenes.flat_gaussians, the same views.
Each workload runs two trainers from the same parameters, antialiasing off and on, alternated --runs times over --steps
iterations each, with CUDA events around the iterations and a device synchronisation at the end.  Reported per arm: median
ms per iteration and the spread (min-max) of the runs, and library launches per iteration.
  bench    with --parent DIR (a checkout of the parent commit, built): bench.py --gpus 1 --steps --bench_steps --warmup 10
           --no-comparators --no-cpu-baseline run --rounds times in this tree and in DIR, alternating: ms per step and GPU
           launches per 100 steps of each.
The card's name and power limit are printed in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gms_b200 import _lib, scenes  # noqa: E402
from gms_b200.model import FreeGaussianModel, MeshGaussianModel  # noqa: E402
from gms_b200.trainer import FreeOptimizationParams, FreeTrainer, MeshTrainer  # noqa: E402

NO_DENSIFY = dict(densify_from_iter=10 ** 9, densify_until_iter=10 ** 9, opacity_reset_interval=10 ** 9, iterations=10 ** 9)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable: {e}"


def views(n, W, H, seed=0):
    g = torch.Generator().manual_seed(seed)
    cams, gts = [], []
    for k, c in enumerate(scenes.ring_cameras(n, 3.2, W, H, elevation_deg=20.0)):
        c.uid = ("view", k)
        cams.append(c.to("cuda"))
        gts.append(torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8).cuda())
    return cams, gts


def time_arm(trainer, cams, gts, steps, first):
    """(ms per iteration, library launches per iteration) over `steps` iterations from view `first` on."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    _lib.launch_count(reset=True)
    e0.record()
    for s in range(steps):
        v = (first + s) % len(cams)
        trainer.step(cams[v], gts[v])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, _lib.launch_count(reset=True) / steps


def trainers(workload, faces, P_free):
    bg = torch.zeros(3, device="cuda")
    if workload == "gs_mesh":
        params = scenes.init_mesh_gaussians(*scenes.object_mesh(faces), K=5, seed=3)
        make = lambda aa: MeshTrainer(MeshGaussianModel.from_params(params, "cuda", packed_features=True, active_sh_degree=3), bg,
                                      native=True, antialiasing=aa)
    else:
        g = scenes.flat_gaussians(P_free, 0)
        raw = (g["means3D"], torch.log(g["scales"][:, 1:]).contiguous(), g["rotations"], g["shs"], torch.logit(g["opacities"]))
        make = lambda aa: FreeTrainer(FreeGaussianModel(*raw, "gs_flat", "cuda", 3), bg, 1.0, FreeOptimizationParams(**NO_DENSIFY),
                                      antialiasing=aa)
    return {"off": make(False), "on": make(True)}


def bench_round(tree, steps):
    r = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", "10", "--no-comparators",
                        "--no-cpu-baseline"], cwd=tree, capture_output=True, text=True, check=True)
    line = json.loads([x for x in r.stdout.splitlines() if x.startswith("{")][-1])
    return {"ms_per_step": line["ms_per_step"], "launches_per_100_steps": line["gpu_launches"] * 100.0 / steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--faces", type=int, default=200_000)
    ap.add_argument("--free", type=int, default=1_000_000, help="gs_flat Gaussians")
    ap.add_argument("--views", type=int, default=16)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bench_steps", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not a.bench:
        ap.error("nothing to do without --bench")
    if not torch.cuda.is_available():
        raise RuntimeError("train_antialiasing_eval.py --bench needs a CUDA device")
    print(card())
    cams, gts = views(a.views, 1920, 1080)
    res = {"card": card(), "time_ms": {}, "launches_per_iteration": {}}
    for workload in ("gs_mesh", "gs_flat"):
        arms = trainers(workload, a.faces, a.free)
        for tr in arms.values():
            time_arm(tr, cams, gts, 2 * a.views, 0)         # warm-up: every view learned and seen twice
        t = {k: [] for k in arms}
        launches = {}
        for r in range(a.runs):
            for k, tr in arms.items():
                ms, launches[k] = time_arm(tr, cams, gts, a.steps, r * a.steps)
                t[k].append(ms)
        for k in arms:
            fr = arms[k]._frame if workload == "gs_mesh" else arms[k].frame
            print(f"{workload:8s} antialiasing {k:3s}: ms/iteration median {np.median(t[k]):.3f} [{min(t[k]):.3f}-{max(t[k]):.3f}], "
                  f"launches/iteration {launches[k]:.1f}, overflows {fr.overflows}")
        res["time_ms"][workload] = t
        res["launches_per_iteration"][workload] = launches
        del arms
        torch.cuda.empty_cache()
    if a.parent:
        res["bench"] = {"this": [], "parent": []}
        for _ in range(a.rounds):
            for k, tree in (("this", ROOT), ("parent", a.parent)):
                res["bench"][k].append(bench_round(tree, a.bench_steps))
        for k, rows in res["bench"].items():
            ms = [x["ms_per_step"] for x in rows]
            print(f"bench.py {k:6s} ms/step {[round(x, 3) for x in ms]} launches/100 steps {[x['launches_per_100_steps'] for x in rows]}")
    print(card())
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
