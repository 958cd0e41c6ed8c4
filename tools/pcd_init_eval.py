"""Exactness and timings of the point-cloud initialisation (gms_knn_dist2, FreeGaussianModel.from_point_cloud).

    python tools/pcd_init_eval.py --check               # 100k uniform and 1M clustered against tests/knn_oracle.py, bit for bit
    python tools/pcd_init_eval.py --bench [--runs 3] [--aten 100k,1m,4m]   # timings, with the card's name, power limit, SM clock

Clouds: the reference's random NeRF-synthetic cloud (scenes.random_point_cloud, 100k uniform in [-1.3, 1.3]^3) and points
sampled on scenes.object_mesh surfaces (knn_oracle.surface_points: clustered on 2D surfaces, as COLMAP clouds are), 1M and 4M.
Arms, alternated `--runs` times after a warm-up call of each, CUDA events around each call:
  native   knn.mean_dist2 (gms_knn_dist2: Morton sort, box bounds, pruned exact search; scratch from the caching allocator)
  aten     what a user without simple-knn would write: torch.cdist over chunks of query rows + topk(4, largest=False), the
           mean of the three non-self squared distances (not exact: cdist's matrix-product form rounds differently).
The all-pairs baseline at 4M points reads and writes 16e12 distances (about five minutes on an H100): it is timed in one run
(--runs does not repeat it), and --aten picks the clouds that get the baseline at all.
from_point_cloud is timed with a host clock around the call and a device synchronisation (it includes the host-to-device
copy of the cloud and the one finiteness read-back)."""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import knn_oracle as K  # noqa: E402
from gms_b200 import knn, scenes  # noqa: E402
from gms_b200.model import FreeGaussianModel  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable: {e}"


def clouds(sizes):
    out = {}
    if "100k" in sizes:
        out["100k uniform"] = scenes.random_point_cloud(100_000, 0)[0]
    if "1m" in sizes:
        out["1M clustered"] = K.surface_points(1_000_000, seed=1)
    if "4m" in sizes:
        out["4M clustered"] = K.surface_points(4_000_000, seed=2)
    return out


def aten_knn(pts: torch.Tensor, chunk: int) -> torch.Tensor:
    out = torch.empty(pts.shape[0], device=pts.device)
    for s in range(0, pts.shape[0], chunk):
        d = torch.cdist(pts[s:s + chunk], pts)
        v = torch.topk(d, 4, dim=1, largest=False).values[:, 1:]
        out[s:s + chunk] = (v * v).mean(dim=1)
    return out


def timed(fn, *a):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn(*a)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def check():
    ok = True
    for name, pts in clouds(("100k", "1m")).items():
        got = knn.mean_dist2(torch.from_numpy(pts).cuda()).cpu().numpy()
        ref, fb = K.dist2(pts, return_fallbacks=True)
        bad = int((got.view(np.uint32) != ref.view(np.uint32)).sum())
        print(f"check {name}: {bad} of {pts.shape[0]} rows differ from the oracle ({fb} oracle rows by brute force)")
        ok = ok and bad == 0
    return ok


def bench(runs: int, aten_sizes):
    print(card())
    for (key, name), pts_np in zip((("100k", "100k uniform"), ("1m", "1M clustered"), ("4m", "4M clustered")),
                                   clouds(("100k", "1m", "4m")).values()):
        pts = torch.from_numpy(pts_np).cuda()
        P = pts.shape[0]
        chunk = max(256, min(4096, int(2 ** 32 // P)))         # <= 16 GB of distances per chunk
        aten = key in aten_sizes
        knn.mean_dist2(pts)
        if aten:
            aten_knn(pts[:min(P, 2 * chunk)], chunk)            # warm-up of cdist / topk at this chunk shape
        nat, ate = [], []
        for r in range(runs):
            nat.append(timed(knn.mean_dist2, pts))
            if aten and (r == 0 or P <= 1_000_000):
                ate.append(timed(aten_knn, pts, chunk))
        nat.append(timed(knn.mean_dist2, pts))
        line = f"{name}: native gms_knn_dist2 ms {', '.join(f'{x:.2f}' for x in nat)}"
        if ate:
            line += (f" | aten cdist+topk (chunk {chunk}) ms {', '.join(f'{x:.1f}' for x in ate)} | "
                     f"speed-up {np.median(ate) / np.median(nat):.0f}x")
        print(line)
        if P <= 1_000_000:
            colors = np.full(pts_np.shape, 0.5)
            FreeGaussianModel.from_point_cloud(pts_np, colors, "gs_flat")
            ts = []
            for _ in range(runs):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                FreeGaussianModel.from_point_cloud(pts_np, colors, "gs_flat")
                torch.cuda.synchronize()
                ts.append(1e3 * (time.perf_counter() - t0))
            print(f"{name}: from_point_cloud (gs_flat) ms {', '.join(f'{x:.1f}' for x in ts)}")
        del pts
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--aten", default="100k,1m,4m", help="clouds that also time the cdist + topk baseline")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("pcd_init_eval needs a CUDA device")
    ok = check() if a.check else True
    if a.bench:
        bench(a.runs, a.aten.split(","))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
