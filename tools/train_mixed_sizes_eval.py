"""Training on views of different sizes: what one frame sized for the largest view costs.

    python tools/train_mixed_sizes_eval.py --bench [--parent DIR] [--out FILE]

Model: scenes.object_mesh(--faces) at K = 5 (1M mesh-Gaussians at the default 200k faces), trained by MeshTrainer (native,
Adam on).  Views: --views ring cameras; ground truth: seeded uint8 noise of each view's size.
  time    per-iteration time of two arms, --runs alternating runs of --steps iterations each, CUDA events around the
          iterations and a device synchronisation at the end: "mixed" alternates 1920x1080 and 1080x1920 views through one
          frame sized for 1920x1920; "uniform" runs the same cameras all at 1920x1080 through a 1920x1080 frame.
  memory  the device memory one 1920x1920 frame holds after running both sizes (workspace + the rasterizer's grow-only
          scratch), against one exact-size frame per size, measured as torch.cuda.memory_allocated deltas, with the
          workspace byte counts gms_frame_workspace_bytes gives.
  bench   with --parent DIR (a checkout of the parent commit, built): bench.py --gpus 1 --steps --bench_steps --warmup 10
          --no-comparators --no-cpu-baseline (the bare trainer loop) run --rounds times in this tree and in DIR,
          alternating: ms per step and GPU launches per 100 steps of each.
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
from gms_b200.model import MeshGaussianModel  # noqa: E402
from gms_b200.trainer import MeshTrainer, NativeFrame  # noqa: E402

LAND, PORT = (1920, 1080), (1080, 1920)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable: {e}"


def views(n, sizes, seed=0):
    g = torch.Generator().manual_seed(seed)
    cams, gts = [], []
    for k in range(n):
        W, H = sizes[k % len(sizes)]
        c = scenes.ring_cameras(n, 3.2, W, H, elevation_deg=20.0)[k]
        c.uid = ("view", k)
        cams.append(c.to("cuda"))
        gts.append(torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8).cuda())
    return cams, gts


def make_model(params):
    return MeshGaussianModel.from_params(params, "cuda", packed_features=True, active_sh_degree=3)


def time_arm(trainer, cams, gts, steps, first):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for s in range(steps):
        v = (first + s) % len(cams)
        trainer.step(cams[v], gts[v])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def memory(params, mixed_cams, mixed_gts):
    """Device bytes the frames hold after one step on each size: one 1920x1920 up_to frame against one frame per size."""
    bg = torch.zeros(3, device="cuda")
    out = {}
    for arm in ("one_max_size_frame", "frame_per_size"):
        model = make_model(params)
        tr = MeshTrainer(model, bg, native=True, max_size=(1920, 1920))
        tr.optimizer_step = False
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        frames = {}
        for c, g in zip(mixed_cams[:2], mixed_gts[:2]):
            if arm == "frame_per_size":
                size = (c.image_width, c.image_height)
                frames.setdefault(size, NativeFrame(model, *size, sync_free=True))
                tr._frame = frames[size]
            tr.step(c, g)
        torch.cuda.synchronize()
        out[arm] = torch.cuda.memory_allocated() - before
        del tr, model, frames
        torch.cuda.empty_cache()
    P = params._scale.shape[0]
    L = _lib.lib()
    out["workspace_bytes"] = {"1920x1920": int(L.gms_frame_workspace_bytes(P, 1920, 1920)),
                              "1920x1080 + 1080x1920": int(L.gms_frame_workspace_bytes(P, *LAND) + L.gms_frame_workspace_bytes(P, *PORT))}
    return out


def bench_round(tree, steps):
    r = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", "10", "--no-comparators",
                        "--no-cpu-baseline"], cwd=tree,
                       capture_output=True, text=True, check=True)
    line = json.loads([x for x in r.stdout.splitlines() if x.startswith("{")][-1])
    return {"ms_per_step": line["ms_per_step"], "launches_per_100_steps": line["gpu_launches"] * 100.0 / steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--faces", type=int, default=200_000)
    ap.add_argument("--views", type=int, default=16)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bench_steps", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not a.bench:
        ap.error("nothing to do without --bench")
    if not torch.cuda.is_available():
        raise RuntimeError("train_mixed_sizes_eval.py --bench needs a CUDA device")
    print(card())
    verts, faces = scenes.object_mesh(a.faces)
    params = scenes.init_mesh_gaussians(verts, faces, K=5, seed=3)
    bg = torch.zeros(3, device="cuda")
    arms = {"mixed": ((1920, 1920), views(a.views, [LAND, PORT])), "uniform": (LAND, views(a.views, [LAND]))}
    trainers = {k: MeshTrainer(make_model(params), bg, native=True, max_size=m) for k, (m, _) in arms.items()}
    res = {"P": int(params._scale.shape[0]), "card": card(), "time_ms": {k: [] for k in arms}}
    for k, (_, (cams, gts)) in arms.items():
        time_arm(trainers[k], cams, gts, 2 * a.views, 0)        # warm-up: every view learned and seen twice
    for r in range(a.runs):
        for k, (_, (cams, gts)) in arms.items():
            res["time_ms"][k].append(time_arm(trainers[k], cams, gts, a.steps, r * a.steps))
    for k, t in res["time_ms"].items():
        fr = trainers[k]._frame
        print(f"{k:8s} ms/iteration median {np.median(t):.3f} [{min(t):.3f}-{max(t):.3f}]  frame {fr.W}x{fr.H}, overflows {fr.overflows}")
    del trainers
    torch.cuda.empty_cache()
    res["memory"] = memory(params, *arms["mixed"][1])
    m = res["memory"]
    print(f"memory: one 1920x1920 frame {m['one_max_size_frame'] / 2**20:.1f} MiB, one frame per size {m['frame_per_size'] / 2**20:.1f} MiB;"
          f" workspaces {json.dumps({k: round(v / 2**20, 1) for k, v in m['workspace_bytes'].items()})} MiB")
    if a.parent:
        res["bench"] = {"this": [], "parent": []}
        for _ in range(a.rounds):
            for k, tree in (("this", ROOT), ("parent", a.parent)):
                res["bench"][k].append(bench_round(tree, a.bench_steps))
        for k, rows in res["bench"].items():
            ms = [x["ms_per_step"] for x in rows]
            print(f"bench.py {k:6s} ms/step {[round(x, 3) for x in ms]} launches/100 steps {[x['launches_per_100_steps'] for x in rows]}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
