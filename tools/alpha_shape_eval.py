"""Timings of the dummy-mesh path (alpha_shape.alpha_shape + estimate_normals) against the host path a user of open3d's
algorithm would run without it: scipy's Qhull Delaunay plus the vectorised open3d filter (tests/alpha_shape_oracle.py) and
cKDTree normals.

    python tools/alpha_shape_eval.py --bench [--gaussians 300000] [--alphas 0.003,0.01] [--runs 3] [--host-runs 1]

Points: the x2 pseudo-mesh of gs_flat Gaussians laid flat on scenes.object_mesh surfaces (alpha_shape_cases), so the
neighbourhoods resemble a trained model's.  GPU arms are timed with a host clock around the call and a device
synchronisation (alpha_shape synchronises twice itself), alternated `--runs` times after a warm-up call; the host arm runs
`--host-runs` times.  The two triangle sets are compared and the card's name and power limit are printed in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import alpha_shape_cases as cases  # noqa: E402
import alpha_shape_oracle as oracle  # noqa: E402
from gms_b200.alpha_shape import alpha_shape, estimate_normals  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable: {e}"


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--gaussians", type=int, default=300000)
    ap.add_argument("--alphas", default="0.003,0.01")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--host-runs", type=int, default=1)
    args = ap.parse_args()
    if not args.bench:
        ap.error("--bench is the only mode")
    if not torch.cuda.is_available():
        raise SystemExit("alpha_shape_eval: needs a CUDA device (there is no CPU timing path)")
    print(card(), flush=True)
    pts = cases.pseudomesh_points(args.gaussians, seed=0)
    P64 = pts.cpu().numpy().astype(np.float64)
    print(f"{pts.shape[0]} points from {args.gaussians} Gaussians", flush=True)
    results = []
    for alpha in [float(a) for a in args.alphas.split(",")]:
        alpha_shape(pts, alpha), estimate_normals(pts)          # warm-up
        ta, tn = [], []
        for _ in range(args.runs):
            t, (v, f, idx) = timed(lambda: alpha_shape(pts, alpha))
            ta.append(t)
            t, _n = timed(lambda: estimate_normals(pts))
            tn.append(t)
        th = []
        for _ in range(args.host_runs):
            t0 = time.perf_counter()
            ref, _ = oracle.alpha_faces(P64, alpha)
            th_alpha = time.perf_counter() - t0
            t0 = time.perf_counter()
            from scipy.spatial import cKDTree
            cKDTree(P64).query(P64, k=30, distance_upper_bound=0.1)      # the neighbour search of the normals
            th.append((th_alpha, time.perf_counter() - t0))
        got = set(map(tuple, idx.cpu().numpy()[f.cpu().numpy()].tolist()))
        r = dict(alpha=alpha, points=int(pts.shape[0]), faces=len(got), oracle_faces=len(ref), differ=len(got ^ ref),
                 gpu_alpha_ms=[round(1e3 * t, 2) for t in ta], gpu_normals_ms=[round(1e3 * t, 2) for t in tn],
                 host_qhull_filter_s=[round(t[0], 2) for t in th], host_kdtree_query_s=[round(t[1], 2) for t in th])
        r["speedup_alpha"] = round(min(t[0] for t in th) / float(np.median(ta)), 1)
        print(json.dumps(r), flush=True)
        results.append(r)
    return results


if __name__ == "__main__":
    main()
