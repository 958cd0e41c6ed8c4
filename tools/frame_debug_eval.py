"""Debug mode: what the reference's pipe.debug (train.py --debug) costs a native training step.

    python tools/frame_debug_eval.py --bench [--parent DIR] [--out FILE]

Workloads (as tools/train_antialiasing_eval.py): gs_mesh, MeshTrainer (native, Adam on) at 1M mesh-Gaussians, and gs_flat,
FreeTrainer (no densification in the window) at 1M Gaussians, 1920x1080, --views ring cameras, seeded uint8 noise as ground
truth.  Each workload runs two trainers from the same parameters, debug off and on, alternated --runs times over --steps
iterations each.  Reported per arm: median ms per iteration, the spread (min-max) of the runs and library launches per
iteration.  Then, for the debug arm: the host copy of the snapshot (DebugMode.snapshot, timed with a device synchronisation
on either side) per iteration, and, in a run of its own with the library's kernel timers on, the binning check kernels'
time per iteration.  With --parent DIR (a built checkout of the parent commit): bench.py --gpus 1 alternated --rounds times
in this tree and in DIR.  The card's name and power limit are printed in the same run."""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from train_antialiasing_eval import NO_DENSIFY, bench_round, card, np, scenes, time_arm, torch, views  # noqa: E402

from gms_b200 import _lib  # noqa: E402
from gms_b200.model import FreeGaussianModel, MeshGaussianModel  # noqa: E402
from gms_b200.trainer import FreeOptimizationParams, FreeTrainer, MeshTrainer  # noqa: E402


def trainers(workload, faces, P_free, dump):
    bg = torch.zeros(3, device="cuda")
    if workload == "gs_mesh":
        params = scenes.init_mesh_gaussians(*scenes.object_mesh(faces), K=5, seed=3)
        make = lambda on: MeshTrainer(MeshGaussianModel.from_params(params, "cuda", packed_features=True, active_sh_degree=3), bg,
                                      native=True, debug=on, debug_snapshot=dump)
    else:
        g = scenes.flat_gaussians(P_free, 0)
        raw = (g["means3D"], torch.log(g["scales"][:, 1:]).contiguous(), g["rotations"], g["shs"], torch.logit(g["opacities"]))
        make = lambda on: FreeTrainer(FreeGaussianModel(*raw, "gs_flat", "cuda", 3), bg, 1.0, FreeOptimizationParams(**NO_DENSIFY),
                                      debug=on, debug_snapshot=dump)
    return {"off": make(False), "on": make(True)}


def snapshot_ms(tr, cams, gts, reps):
    """ms of one DebugMode.snapshot (the host copy a debug step takes before its frame)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for r in range(reps):
        tr._debug.snapshot(tr, cams[r % len(cams)], gts[r % len(cams)], tr.bg, tr.iteration + 1)
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--faces", type=int, default=200_000)
    ap.add_argument("--free", type=int, default=1_000_000, help="gs_flat Gaussians")
    ap.add_argument("--views", type=int, default=16)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bench_steps", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not a.bench:
        ap.error("nothing to do without --bench")
    if not torch.cuda.is_available():
        raise RuntimeError("frame_debug_eval.py --bench needs a CUDA device")
    print(card())
    W, H = 1920, 1080
    cams, gts = views(a.views, W, H)
    res = {"card": card(), "time_ms": {}, "launches_per_iteration": {}, "snapshot_ms": {}, "check_ms": {}}
    dump = os.path.join(tempfile.mkdtemp(), "snapshot_frame.dump")      # written only by a failing step
    for workload in ("gs_mesh", "gs_flat"):
        arms = trainers(workload, a.faces, a.free, dump)
        for tr in arms.values():
            time_arm(tr, cams, gts, 2 * a.views, 0)         # warm-up: every view learned and seen twice
        t = {k: [] for k in arms}
        launches = {}
        for r in range(a.runs):
            for k, tr in arms.items():
                ms, launches[k] = time_arm(tr, cams, gts, a.steps, r * a.steps)
                t[k].append(ms)
        for k in arms:
            print(f"{workload:8s} debug {k:3s}: ms/iteration median {np.median(t[k]):.3f} [{min(t[k]):.3f}-{max(t[k]):.3f}], "
                  f"launches/iteration {launches[k]:.1f}")
        snap = snapshot_ms(arms["on"], cams, gts, 8)
        _lib.set_option("time_kernels", 1)
        _lib.kernel_times(reset=True)
        time_arm(arms["on"], cams, gts, a.views, 0)
        kt = _lib.kernel_times(reset=True)
        _lib.set_option("time_kernels", 0)
        chk_ms, chk_n = kt.get("debug_check", (0.0, 0))
        on = float(np.median(t["on"]))
        print(f"{workload:8s} snapshot copy: {snap:.3f} ms per iteration ({100 * snap / on:.1f} % of a debug iteration); "
              f"binning check kernels: {chk_ms / a.views:.3f} ms per iteration over {chk_n / a.views:.0f} launches")
        res["time_ms"][workload] = t
        res["launches_per_iteration"][workload] = launches
        res["snapshot_ms"][workload] = snap
        res["check_ms"][workload] = chk_ms / a.views
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
