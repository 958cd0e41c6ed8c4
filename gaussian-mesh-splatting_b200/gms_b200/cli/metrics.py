"""python -m gms_b200.cli.metrics -m <output> [<output> ...] [--gs_type gs_flat] [--lpips [--lpips_weights DIR]]: the
reference's metrics.py on the device.

For every method directory test/<method>/ of every model directory, renders_{gs_type}/ is paired with gt/ by file name in
os.listdir order.  The PNGs are decoded on the host, uploaded, turned into byte / 255 (gms_image_dequantize) and scored by
gms_image_metrics, all on one stream with one host synchronisation per method: SSIM, and the PSNR over all channels of the
[1,3,H,W] batch as metrics.py computes it.  results_{gs_type}.json and per_view_{gs_type}.json have the reference's shape;
per-view values are rounded to float32 as the reference's tensors hold them, means are the float32 mean of those.

With --lpips, every pair is also scored by gms_lpips_vgg (gms_b200.lpips, VGG16 LPIPS v0.1 as metrics.py:74 computes it) in
the same stream pass, and "LPIPS" follows "SSIM" and "PSNR" in both files and in the printed means.  The weights are read
from --lpips_weights (default: <torch.hub.get_dir()>/checkpoints, where a run of the reference leaves vgg16-397923af.pth and
vgg.pth); this project neither ships nor downloads them.  Without --lpips there is no LPIPS key."""
from __future__ import annotations

import json
import os
import sys
from argparse import ArgumentParser
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import torch

from .. import dataset, io_image
from ..lpips import Lpips
from ..metrics import METRIC_NAMES, image_metrics, scratch_bytes

SSIM, PSNR = METRIC_NAMES.index("ssim"), METRIC_NAMES.index("psnr")


def read_rgb(path: str) -> np.ndarray:
    """uint8 [H,W,3]: the file's first three channels (to_tensor(...)[:, :3]); a grey image is repeated to three."""
    arr = dataset.decode_image(path, "RGBA")
    return np.ascontiguousarray(arr[..., :3])


def score_method(renders_dir: Path, gt_dir: Path, device, lpips=None) -> tuple:
    """(image names, per-view float64 [n,4] METRIC_NAMES) of one method directory, one synchronisation; given an
    lpips.Lpips, (image names, per-view [n,4], per-view LPIPS float32 [n])."""
    names = os.listdir(renders_dir)
    out = torch.empty(len(names), len(METRIC_NAMES), dtype=torch.float64, device=device)
    lp = torch.empty(len(names), 6, dtype=torch.float32, device=device) if lpips is not None else None
    scratch = None
    bufs = {}
    with ThreadPoolExecutor(max(2, min(8, os.cpu_count() or 2))) as ex:
        pairs = [(ex.submit(read_rgb, str(renders_dir / n)), ex.submit(read_rgb, str(gt_dir / n))) for n in names]
        for k, (fr, fg) in enumerate(pairs):
            r, g = fr.result(), fg.result()
            if r.shape != g.shape:
                raise ValueError(f"{renders_dir / names[k]} is {r.shape[1]}x{r.shape[0]} but its ground truth {g.shape[1]}x{g.shape[0]}")
            H, W, _ = r.shape
            if (H, W) not in bufs:
                bufs[(H, W)] = (torch.empty(3, H, W, dtype=torch.float32, device=device),
                                torch.empty(3, H, W, dtype=torch.float32, device=device))
            rf, gf = bufs[(H, W)]
            need = scratch_bytes(3, H, W)
            if scratch is None or scratch.numel() < need:
                scratch = torch.empty(need, dtype=torch.uint8, device=device)
            io_image.to_device_float(torch.from_numpy(r).pin_memory().to(device, non_blocking=True), out=rf)
            io_image.to_device_float(torch.from_numpy(g).pin_memory().to(device, non_blocking=True), out=gf)
            image_metrics(rf, gf, "training_report", out=out[k], scratch=scratch)
            if lp is not None:
                lpips.lpips(rf, gf, out=lp[k])
    if lp is None:
        return names, out.cpu()
    lp_host = torch.empty(len(names), dtype=torch.float32).pin_memory()
    lp_host.copy_(lp[:, 5], non_blocking=True)          # ordered before the read-back below, which waits for it
    return names, out.cpu(), lp_host


def evaluate(gs_type: str, model_paths, device="cuda", quiet: bool = False, score=score_method, lpips=None) -> dict:
    """metrics.py's evaluate: writes the two JSON files per model directory and returns {model: results}.  Without `lpips`,
    score(renders_dir, gt_dir, device) -> (names, per-view [n,4]) and there is no LPIPS key; given an lpips.Lpips,
    score(renders_dir, gt_dir, device, lpips) -> (names, per-view [n,4], per-view LPIPS [n]).  score is score_method unless
    a test replaces it."""
    results = {}
    for scene_dir in model_paths:
        if not quiet:
            print("Scene:", scene_dir)
        full, per_view = {}, {}
        test_dir = Path(scene_dir) / "test"
        for method in os.listdir(test_dir):
            if not quiet:
                print("Method:", method)
            method_dir = test_dir / method
            if lpips is None:
                names, pv = score(method_dir / f"renders_{gs_type}", method_dir / "gt", device)
            else:
                names, pv, lp = score(method_dir / f"renders_{gs_type}", method_dir / "gt", device, lpips)
            ssims = torch.tensor(pv[:, SSIM].tolist(), dtype=torch.float32)
            psnrs = torch.tensor(pv[:, PSNR].tolist(), dtype=torch.float32)
            lpipss = torch.tensor(torch.as_tensor(lp).tolist(), dtype=torch.float32) if lpips is not None else None
            if not quiet:
                print("  SSIM : {:>12.7f}".format(ssims.mean()))
                print("  PSNR : {:>12.7f}".format(psnrs.mean()))
                if lpipss is not None:
                    print("  LPIPS: {:>12.7f}".format(lpipss.mean()))
                print("")
            full[method] = {"SSIM": ssims.mean().item(), "PSNR": psnrs.mean().item()}
            per_view[method] = {"SSIM": dict(zip(names, ssims.tolist())), "PSNR": dict(zip(names, psnrs.tolist()))}
            if lpipss is not None:
                full[method]["LPIPS"] = lpipss.mean().item()
                per_view[method]["LPIPS"] = dict(zip(names, lpipss.tolist()))
        with open(scene_dir + f"/results_{gs_type}.json", "w") as fp:
            json.dump(full, fp, indent=True)
        with open(scene_dir + f"/per_view_{gs_type}.json", "w") as fp:
            json.dump(per_view, fp, indent=True)
        results[scene_dir] = {"results": full, "per_view": per_view}
    return results


def main(argv=None) -> dict:
    parser = ArgumentParser(description="Metrics script parameters")
    parser.add_argument("--model_paths", "-m", required=True, nargs="+", type=str, default=[])
    parser.add_argument("--gs_type", type=str, default="gs_flat")
    parser.add_argument("--quiet", action="store_true")
    parser.add_argument("--lpips", action="store_true", help="also report LPIPS (VGG16, v0.1) from weights already on disk")
    parser.add_argument("--lpips_weights", type=str, default=None,
                        help="directory holding vgg16-397923af.pth and vgg.pth (default: <torch hub dir>/checkpoints)")
    args = parser.parse_args(sys.argv[1:] if argv is None else argv)
    if not torch.cuda.is_available():
        raise RuntimeError("gms_b200.cli.metrics needs a CUDA device")
    scorer = Lpips.from_cache(args.lpips_weights, device="cuda") if args.lpips else None
    return evaluate(args.gs_type, args.model_paths, quiet=args.quiet, lpips=scorer)


if __name__ == "__main__":
    main()
