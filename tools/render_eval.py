"""Render and evaluation timings on the GPU: the autograd-shim path against the native render frame and view metrics.

    python tools/render_eval.py [--runs 5] [--frames 100] [--views 16] > render_eval.txt

1. Animated sweep, BASELINE config 5 (500k mesh-Gaussians, 1080p; what `bench.py --mode render_animated` times): per frame the
   vertices move by transform_hotdog_fly(t) and the frame is rendered, by trainer.render_frame (shim: one blocking 4-byte
   read-back of N per frame) or by NativeRenderer.render (sync-free after the first frame).  The arms alternate, `--runs`
   runs each, CUDA events over `--frames` timed frames after a warm-up; ms per frame, launches per frame, N, and the largest
   image difference between the arms on the same frame.
2. Evaluation of `--views` views at 1M mesh-Gaussians, 1080p: the reference protocol (render_frame, clamp, ATen L1 / psnr /
   ssim, `.item()` per view, train.py:197-214 + metrics.py:72-73) against NativeRenderer.evaluate (one synchronisation),
   ms per view and both metric sets side by side.
The card's name, power limit and SM clock are read in the same run (nvidia-smi, read-only query)."""
import argparse
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import aten_reference  # noqa: E402
import bench  # noqa: E402
from gms_b200 import _lib, scenes  # noqa: E402
from gms_b200.model import MeshGaussianModel  # noqa: E402
from gms_b200.render import NativeRenderer  # noqa: E402
from gms_b200.trainer import render_frame  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable: {e}"


def sweep(args, dev):
    params, cams, (F, K, W, H) = bench.build_scene("gs_mesh_500k_1080p")
    model = MeshGaussianModel.from_params(params, dev, packed_features=True)
    bg = torch.ones(3, device=dev)
    cams = [c.to(dev) for c in cams]
    ts = torch.linspace(0, 10 * math.pi, 800)
    v0 = model.vertices.detach().clone()
    native = NativeRenderer(model, W, H)
    arms = {"render_frame": lambda cam: render_frame(model, cam, bg)[0],
            "NativeRenderer": lambda cam: native.render(cam, bg)[0]}

    def frame(arm, i):
        with torch.no_grad():
            model.vertices.data.copy_(scenes.transform_hotdog_fly(v0, float(ts[i % len(ts)])))
            return arms[arm](cams[i % len(cams)])

    for arm in arms:                                    # warm-up: every camera twice, both arms
        for i in range(2 * len(cams)):
            frame(arm, i)
    torch.cuda.synchronize()
    res = {arm: [] for arm in arms}
    for run in range(args.runs):
        for arm in arms:
            _lib.launch_count(reset=True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.frames):
                frame(arm, 7 * run + i)
            e1.record()
            torch.cuda.synchronize()
            res[arm].append((e0.elapsed_time(e1) / args.frames, _lib.launch_count(reset=True) / args.frames))
    diff = 0.0
    for i in range(0, 2 * len(cams), 3):
        a = frame("render_frame", i).clone()
        b = frame("NativeRenderer", i)
        diff = max(diff, float((a - b).abs().max()))
    from gms_b200 import rasterizer
    print(f"== animated sweep, config 5: P = {F * K}, {W}x{H}, {args.runs} alternating runs x {args.frames} frames")
    for arm, rs in res.items():
        ms = [r[0] for r in rs]
        print(f"  {arm:15s} ms/frame {np.mean(ms):.3f} (runs {', '.join(f'{m:.3f}' for m in ms)}), launches/frame {rs[-1][1]:.1f}")
    print(f"  N (last frame): shim {rasterizer.last_num_rendered}, native {native.last_num_rendered}; native overflows {native.overflows}")
    print(f"  max |image(render_frame) - image(NativeRenderer)| on the same frame: {diff:.3e}")


def reference_protocol(model, cams, gts, bg):
    """train.py:197-214 (clamp, l1_loss, psnr on [C,H,W]) and metrics.py:72-73 (ssim, psnr on [1,C,H,W]), .item() per view."""
    rows = []
    for cam, gt in zip(cams, gts):
        with torch.no_grad():
            image = torch.clamp(render_frame(model, cam, bg)[0], 0.0, 1.0)
            g = torch.clamp(gt, 0.0, 1.0)
            d2 = (image - g) ** 2
            l1 = aten_reference.l1_loss(image, g).item()
            ss = aten_reference.ssim(image[None], g[None]).item()
            psnr_all = (20 * torch.log10(1.0 / torch.sqrt(d2.reshape(1, -1).mean(1)))).item()
            psnr_pc = (20 * torch.log10(1.0 / torch.sqrt(d2.reshape(3, -1).mean(1)))).mean().item()
        rows.append([l1, ss, psnr_all, psnr_pc])
    return np.array(rows)


def evaluation(args, dev):
    params, cams, (F, K, W, H) = bench.build_scene("gs_mesh_1M_1080p")
    model = MeshGaussianModel.from_params(params, dev, packed_features=True)
    bg = torch.ones(3, device=dev)
    cams = [cams[i % len(cams)].to(dev) for i in range(args.views)]
    g = torch.Generator(device=dev).manual_seed(0)
    with torch.no_grad():       # ground truth: the render plus noise, so that the scores are those of a decent model
        gts = [(render_frame(model, c, bg)[0] + 0.03 * torch.randn(3, H, W, generator=g, device=dev)).clamp(0, 1).contiguous() for c in cams]
    native = NativeRenderer(model, W, H)
    native.evaluate(cams, gts, bg)              # warm-up (and every view's N)
    reference_protocol(model, cams[:2], gts[:2], bg)
    t_ref, t_nat = [], []
    for _ in range(args.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ref = reference_protocol(model, cams, gts, bg)
        t_ref.append((time.perf_counter() - t0) * 1e3 / len(cams))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = native.evaluate(cams, gts, bg)
        t_nat.append((time.perf_counter() - t0) * 1e3 / len(cams))
    print(f"== evaluation: P = {F * K}, {W}x{H}, {len(cams)} views, {args.runs} alternating runs (host clock, each ends in a sync)")
    print(f"  reference protocol ms/view {np.mean(t_ref):.3f} (runs {', '.join(f'{t:.3f}' for t in t_ref)})")
    print(f"  evaluate()         ms/view {np.mean(t_nat):.3f} (runs {', '.join(f'{t:.3f}' for t in t_nat)}); re-ran views {res.rerun}")
    nat = res.per_view.numpy()
    print("  view | L1 ref / native | SSIM ref / native | PSNR(all) ref / native | PSNR(per channel) ref / native")
    for v in range(len(cams)):
        print(f"  {v:4d} | {ref[v, 0]:.7f} / {nat[v, 0]:.7f} | {ref[v, 1]:.7f} / {nat[v, 1]:.7f} | "
              f"{ref[v, 2]:.5f} / {nat[v, 2]:.5f} | {ref[v, 3]:.5f} / {nat[v, 3]:.5f}")
    print(f"  mean | {ref[:, 0].mean():.7f} / {nat[:, 0].mean():.7f} | {ref[:, 1].mean():.7f} / {nat[:, 1].mean():.7f} | "
          f"{ref[:, 2].mean():.5f} / {nat[:, 2].mean():.5f} | {ref[:, 3].mean():.5f} / {nat[:, 3].mean():.5f}")
    print(f"  largest |ref - native| per column: {np.abs(ref - nat).max(0)}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--views", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_eval.py measures on the GPU; no CUDA device found")
    print(card())
    dev = torch.device("cuda", 0)
    sweep(args, dev)
    evaluation(args, dev)
    print(card())


if __name__ == "__main__":
    main()
