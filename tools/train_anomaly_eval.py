"""Anomaly detection: what the reference's train.py --detect_anomaly costs a native training step, and how close the NaN scan
comes to the HBM floor.

    python tools/train_anomaly_eval.py --bench [--parent DIR] [--out FILE]

Workloads (as tools/train_antialiasing_eval.py):
  gs_mesh  MeshTrainer (native, Adam on): scenes.object_mesh(--faces) at K = 5 (1M mesh-Gaussians at the default 200k faces),
           1920x1080, --views ring cameras, seeded uint8 noise as ground truth.
  gs_flat  FreeTrainer (no densification in the window): 1M scenes.flat_gaussians, the same views.
Each workload runs two trainers from the same parameters, detect_anomaly off and on, alternated --runs times over --steps
iterations each, with CUDA events around the iterations and a device synchronisation at the end.  Reported per arm: median
ms per iteration, the spread (min-max) of the runs and library launches per iteration.  Then, in a run of its own with the
library's kernel timers on, the flagged arm's nan_scan time per iteration and its achieved bandwidth, from the bytes each
stage scans (computed from the shapes below), against the H100 SXM's 3.35 TB/s.
  scan     gms_nan_scan alone over one clean 256 MiB buffer, --scan_reps launches between two events: time and GB/s.
  bench    with --parent DIR (a checkout of the parent commit, built): bench.py --gpus 1 --steps --bench_steps --warmup 10
           --no-comparators --no-cpu-baseline run --rounds times in this tree and in DIR, alternating.
The card's name and power limit are printed in the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from train_antialiasing_eval import NO_DENSIFY, bench_round, card, np, scenes, time_arm, torch, views  # noqa: E402

from gms_b200 import _lib, anomaly  # noqa: E402
from gms_b200.model import FreeGaussianModel, MeshGaussianModel  # noqa: E402
from gms_b200.trainer import FreeOptimizationParams, FreeTrainer, MeshTrainer  # noqa: E402

HBM = 3.35e12


def trainers(workload, faces, P_free):
    bg = torch.zeros(3, device="cuda")
    if workload == "gs_mesh":
        params = scenes.init_mesh_gaussians(*scenes.object_mesh(faces), K=5, seed=3)
        make = lambda on: MeshTrainer(MeshGaussianModel.from_params(params, "cuda", packed_features=True, active_sh_degree=3), bg,
                                      native=True, detect_anomaly=on)
    else:
        g = scenes.flat_gaussians(P_free, 0)
        raw = (g["means3D"], torch.log(g["scales"][:, 1:]).contiguous(), g["rotations"], g["shs"], torch.logit(g["opacities"]))
        make = lambda on: FreeTrainer(FreeGaussianModel(*raw, "gs_flat", "cuda", 3), bg, 1.0, FreeOptimizationParams(**NO_DENSIFY),
                                      detect_anomaly=on)
    return {"off": make(False), "on": make(True)}


def scanned_bytes(workload, tr, W, H):
    """Bytes the flagged frame scans per iteration: dL/dimage; the gradient records (12 floats per Gaussian); the preprocess
    outputs (dmeans3D 3, dscales 3, drotations 4, dopacity 1, and the colour gradient 3 (mesh: the factored path) or the SH
    rows 3M (gs_flat: the dense path)); d_vertices, d_alpha_raw, d_scale_raw (mesh) or d_scaling_raw, d_rotation_raw, accum."""
    m = tr.model
    P = m._scale.shape[0] if workload == "gs_mesh" else m.P
    sh = 3 if workload == "gs_mesh" else 3 * m._features.shape[1]
    last = 3 * m.vertices.shape[0] + 4 * P if workload == "gs_mesh" else (m.scale_cols + 4 + 1) * P
    return 4 * (3 * W * H + 12 * P + (11 + sh) * P + last)


def scan_alone(reps):
    x = torch.zeros(64 << 20, device="cuda")
    rec = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    for _ in range(3):
        anomaly.nan_scan(rec, 0, [(0, x)])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        anomaly.nan_scan(rec, 0, [(0, x)])
    e1.record()
    torch.cuda.synchronize()
    assert int(rec.item()) == -1
    ms = e0.elapsed_time(e1) / reps
    return ms, x.numel() * 4 / (ms * 1e-3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--faces", type=int, default=200_000)
    ap.add_argument("--free", type=int, default=1_000_000, help="gs_flat Gaussians")
    ap.add_argument("--views", type=int, default=16)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--scan_reps", type=int, default=200)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bench_steps", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not a.bench:
        ap.error("nothing to do without --bench")
    if not torch.cuda.is_available():
        raise RuntimeError("train_anomaly_eval.py --bench needs a CUDA device")
    print(card())
    W, H = 1920, 1080
    cams, gts = views(a.views, W, H)
    res = {"card": card(), "time_ms": {}, "launches_per_iteration": {}, "nan_scan": {}}
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
            print(f"{workload:8s} detect_anomaly {k:3s}: ms/iteration median {np.median(t[k]):.3f} [{min(t[k]):.3f}-{max(t[k]):.3f}], "
                  f"launches/iteration {launches[k]:.1f}, overflows {fr.overflows}")
        _lib.set_option("time_kernels", 1)
        _lib.kernel_times(reset=True)
        time_arm(arms["on"], cams, gts, a.views, 0)
        kt = _lib.kernel_times(reset=True)
        _lib.set_option("time_kernels", 0)
        scan_ms, scans = kt.get("nan_scan", (0.0, 0))
        nbytes = scanned_bytes(workload, arms["on"], W, H)
        per_it = scan_ms / a.views
        bw = nbytes / (per_it * 1e-3) if per_it > 0 else 0.0
        print(f"{workload:8s} nan_scan: {per_it:.3f} ms per iteration over {scans / a.views:.0f} launches, {nbytes / 1e6:.1f} MB scanned, "
              f"{bw / 1e9:.0f} GB/s ({100 * bw / HBM:.0f} % of 3.35 TB/s)")
        res["time_ms"][workload] = t
        res["launches_per_iteration"][workload] = launches
        res["nan_scan"][workload] = {"ms_per_iteration": per_it, "bytes": nbytes, "GBps": bw / 1e9}
        del arms
        torch.cuda.empty_cache()
    ms, bw = scan_alone(a.scan_reps)
    print(f"nan_scan alone, 256 MiB clean: {ms:.3f} ms, {bw / 1e9:.0f} GB/s ({100 * bw / HBM:.0f} % of 3.35 TB/s)")
    res["nan_scan"]["alone_256MiB"] = {"ms": ms, "GBps": bw / 1e9}
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
