"""gs_points (pseudo-mesh) render and evaluation timings on the GPU: the autograd-shim path against PointsRenderer.

    python tools/points_render_eval.py [--runs 5] [--frames 100] [--views 16] > points_render_eval.txt

Model: BASELINE config 5 (100k faces x 5 mesh-Gaussians) turned into its 500k-triangle pseudo-mesh by
points_prepare_vertices (PointsModel.from_gaussians of the expansion's raw xyz / _scaling / _rotation), rendered at 1080p.
1. Animated sweep (scripts/render_points_time_animated.py): per frame the triangles move by transform_hotdog(t),
   t = linspace(0, 10 pi, frames), and the frame is rendered by render_points_frame (shim: points_prepare_scaling_rot, an
   ATen sigmoid, GaussianRasterizer with its blocking 4-byte read-back of N) or by PointsRenderer.render(triangles=...)
   (sync-free after the first frame).  Both arms pay the same transform_hotdog.  The arms alternate, `--runs` runs each,
   CUDA events over `--frames` frames after a warm-up: ms per frame, library launches per frame, N, the largest image
   difference between the arms on the same frame, and the expand_fwd span (CUDA events inside the library, separate pass).
2. Evaluation of `--views` views under both protocols: PointsRenderer.evaluate (one synchronisation) against a per-view
   loop of the shim render + ATen L1 / ssim / psnr with `.item()` per view (train.py:197-214; for "metrics", the 8-bit
   round trip of save_image + metrics.py:72-73 first).  ms per view (host clock) and the largest metric difference.
The card's name, power limit and SM clock are read in the same run (nvidia-smi, read-only query)."""
import argparse
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import aten_reference  # noqa: E402
import bench  # noqa: E402
from gms_b200 import _lib, rasterizer, scenes  # noqa: E402
from gms_b200.model import MeshGaussianModel, PointsModel  # noqa: E402
from gms_b200.render import PointsRenderer, render_points_frame  # noqa: E402
from render_eval import card  # noqa: E402


def points_model(dev):
    params, cams, (F, K, W, H) = bench.build_scene("gs_mesh_500k_1080p")
    with torch.no_grad():
        xyz, sl, rr = MeshGaussianModel.from_params(params, dev, packed_features=True).expand_fused(activated=False)
    model = PointsModel.from_gaussians(xyz, sl, rr, params._features_dc, params._features_rest, params._opacity, dev)
    return model, [c.to(dev) for c in cams], W, H


def sweep(args, model, cams, W, H):
    bg = torch.ones(3, device=model.triangles.device)
    ts = torch.linspace(0, 10 * math.pi, args.frames)
    native = PointsRenderer(model, W, H)
    arms = {"render_points_frame": lambda cam, tri: render_points_frame(model, cam, bg, triangles=tri)[0],
            "PointsRenderer": lambda cam, tri: native.render(cam, bg, triangles=tri)[0]}

    def frame(arm, i):
        with torch.no_grad():
            return arms[arm](cams[i % len(cams)], scenes.transform_hotdog(model.triangles, float(ts[i % len(ts)])))

    for arm in arms:                                    # warm-up: every camera twice, both arms
        for i in range(2 * len(cams)):
            frame(arm, i)
    torch.cuda.synchronize()
    warm_overflows = native.overflows
    res = {arm: [] for arm in arms}
    for run in range(args.runs):
        for arm in arms:
            _lib.launch_count(reset=True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.frames):
                frame(arm, i)
            e1.record()
            torch.cuda.synchronize()
            res[arm].append((e0.elapsed_time(e1) / args.frames, _lib.launch_count(reset=True) / args.frames))
    timed_overflows = native.overflows - warm_overflows
    spans = {}
    for arm in arms:
        _lib.set_option("time_kernels", 1)
        _lib.kernel_times(reset=True)
        for i in range(args.frames):
            frame(arm, i)
        torch.cuda.synchronize()
        spans[arm] = _lib.kernel_times(reset=True)
        _lib.set_option("time_kernels", 0)
    diff = 0.0
    for i in range(0, args.frames, 7):
        a = frame("render_points_frame", i).clone()
        b = frame("PointsRenderer", i)
        diff = max(diff, float((a - b).abs().max()))
    print(f"== gs_points animated sweep: P = {model.triangles.shape[0]}, {W}x{H}, transform_hotdog over t = linspace(0, 10 pi, "
          f"{args.frames}), {args.runs} alternating runs x {args.frames} frames")
    for arm, rs in res.items():
        ms = [r[0] for r in rs]
        print(f"  {arm:20s} ms/frame {np.mean(ms):.3f} (runs {', '.join(f'{m:.3f}' for m in ms)}), launches/frame {rs[-1][1]:.1f}")
    print(f"  N (last frame): shim {rasterizer.last_num_rendered}, native {native.last_num_rendered}; native overflows {warm_overflows} in the warm-up, "
          f"{timed_overflows} in the {args.runs * args.frames} timed frames (an overflowed frame renders the background)")
    print(f"  max |image(render_points_frame) - image(PointsRenderer)| on the same frame: {diff:.3e}")
    for arm, kt in spans.items():
        rows = ", ".join(f"{k} {ms / args.frames:.4f}" for k, (ms, n) in kt.items() if n)
        print(f"  {arm} kernel spans, ms/frame: {rows}")


def reference_protocol(model, cams, gts, bg, protocol):
    """Shim render, then train.py:197-214 (clamp, l1_loss, psnr on [C,H,W]) and metrics.py:72-73 (ssim, psnr on
    [1,C,H,W]), `.item()` per view; protocol "metrics" first takes both images through save_image's 8-bit rounding."""
    rows = []
    for cam, gt in zip(cams, gts):
        with torch.no_grad():
            image, g = torch.clamp(render_points_frame(model, cam, bg)[0], 0.0, 1.0), torch.clamp(gt, 0.0, 1.0)
            if protocol == "metrics":
                image, g = ((t.mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8).float() / 255.0) for t in (image, g))
            d2 = (image - g) ** 2
            l1 = aten_reference.l1_loss(image, g).item()
            ss = aten_reference.ssim(image[None], g[None]).item()
            psnr_all = (20 * torch.log10(1.0 / torch.sqrt(d2.reshape(1, -1).mean(1)))).item()
            psnr_pc = (20 * torch.log10(1.0 / torch.sqrt(d2.reshape(3, -1).mean(1)))).mean().item()
        rows.append([l1, ss, psnr_all, psnr_pc])
    return np.array(rows)


def evaluation(args, model, cams, W, H):
    dev = model.triangles.device
    bg = torch.ones(3, device=dev)
    cams = [cams[i % len(cams)] for i in range(args.views)]
    g = torch.Generator(device=dev).manual_seed(0)
    with torch.no_grad():       # ground truth: the render plus noise, so that the scores are those of a decent model
        gts = [(render_points_frame(model, c, bg)[0] + 0.03 * torch.randn(3, H, W, generator=g, device=dev)).clamp(0, 1).contiguous()
               for c in cams]
    native = PointsRenderer(model, W, H)
    for protocol in ("training_report", "metrics"):
        native.evaluate(cams, gts, bg, protocol=protocol)          # warm-up (and every view's N)
        reference_protocol(model, cams[:2], gts[:2], bg, protocol)
        t_ref, t_nat = [], []
        for _ in range(args.runs):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ref = reference_protocol(model, cams, gts, bg, protocol)
            t_ref.append((time.perf_counter() - t0) * 1e3 / len(cams))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = native.evaluate(cams, gts, bg, protocol=protocol)
            t_nat.append((time.perf_counter() - t0) * 1e3 / len(cams))
        nat = res.per_view.numpy()
        print(f"== gs_points evaluation, protocol {protocol}: P = {model.triangles.shape[0]}, {W}x{H}, {len(cams)} views, "
              f"{args.runs} alternating runs (host clock, each ends in a sync)")
        print(f"  shim + ATen per view ms/view {np.mean(t_ref):.3f} (runs {', '.join(f'{t:.3f}' for t in t_ref)})")
        print(f"  evaluate()           ms/view {np.mean(t_nat):.3f} (runs {', '.join(f'{t:.3f}' for t in t_nat)}); re-ran views {res.rerun}")
        print(f"  mean ref   L1 {ref[:, 0].mean():.7f} SSIM {ref[:, 1].mean():.7f} PSNR {ref[:, 2].mean():.5f} / {ref[:, 3].mean():.5f}")
        print(f"  mean native L1 {nat[:, 0].mean():.7f} SSIM {nat[:, 1].mean():.7f} PSNR {nat[:, 2].mean():.5f} / {nat[:, 3].mean():.5f}")
        print(f"  largest |ref - native| per column: {np.abs(ref - nat).max(0)}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--views", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("points_render_eval.py measures on the GPU; no CUDA device found")
    print(card())
    dev = torch.device("cuda", 0)
    model, cams, W, H = points_model(dev)
    sweep(args, model, cams, W, H)
    evaluation(args, model, cams, W, H)
    print(card())


if __name__ == "__main__":
    main()
