"""VGG16 LPIPS per view: the native kernels (gms_lpips_vgg) against PyTorch / cuDNN on the same seeded weights and images.

    python tools/lpips_eval.py --bench [--reps 5] [--iters 10]

Arms, alternated within every repetition after a warm-up of each shape:
  native      Lpips.lpips (split-TF32 tensor-core convs, FP32 accuracy)
  torch_fp32  the float32 restatement (tests/lpips_oracle.py, F.conv2d / cuDNN) with allow_tf32 = False
  torch_tf32  the same with cuDNN's defaults (TF32 convolutions): what the reference runs on Hopper
Each is one view: render and ground truth as one batch of two.  Times are CUDA events over `iters` views; the FLOP count
is 2 * MACs of the 13 convs from the layer shapes.  Prints the card and its power limit from the same process, and one
JSON line per size with the median and range over the repetitions."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")]

import lpips_oracle  # noqa: E402
from gms_b200.lpips import Lpips  # noqa: E402

SIZES = [(800, 800), (1080, 1920)]


def conv_flops(H: int, W: int) -> int:
    """2 * MACs of VGG16's 13 convs up to relu5_3 on a batch of two, with the floor of every pooling."""
    macs, h, w = 0, H, W
    for layer in lpips_oracle.LAYERS:
        if layer[0] == "conv":
            macs += h * w * 9 * layer[2] * layer[3]
        elif layer[0] == "pool":
            h, w = h // 2, w // 2
    return 2 * 2 * macs


def card() -> str:
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def timed(fn, iters: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not args.bench:
        ap.error("nothing to do: pass --bench")
    if not torch.cuda.is_available():
        raise RuntimeError("lpips_eval.py --bench needs a CUDA device")
    with tempfile.TemporaryDirectory() as d:
        _, _, vgg16, lin = lpips_oracle.write_weight_files(d, seed=0)
        L = Lpips.from_cache(d, device="cuda")
    vgg16 = {k: v.cuda() for k, v in vgg16.items()}
    lin = {k: v.cuda() for k, v in lin.items()}
    print(f"card: {card()}")
    tf32_default = torch.backends.cudnn.allow_tf32
    for H, W in SIZES:
        g = torch.Generator(device="cuda").manual_seed(H + W)
        img = torch.rand(3, H, W, generator=g, device="cuda")
        gt = (img + 0.05 * torch.randn(3, H, W, generator=g, device="cuda")).clamp(0, 1)
        out = torch.empty(6, device="cuda")

        def native():
            L.lpips(img, gt, out=out)

        def torch_arm(tf32):
            def run():
                torch.backends.cudnn.allow_tf32 = tf32
                with torch.no_grad():
                    lpips_oracle.lpips(img, gt, vgg16, lin, dtype=torch.float32)
            return run

        arms = {"native": native, "torch_fp32": torch_arm(False), "torch_tf32": torch_arm(True)}
        for fn in arms.values():       # warm-up: modules, cuDNN algorithm choice, allocator
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():
                ms[k].append(timed(fn, args.iters))
        torch.backends.cudnn.allow_tf32 = tf32_default
        flops = conv_flops(H, W)
        res = {"size": f"{W}x{H}", "conv_tflop_per_view": flops / 1e12}
        for k, v in ms.items():
            v = sorted(v)
            med = v[len(v) // 2]
            res[k] = {"ms_median": round(med, 3), "ms_min": round(v[0], 3), "ms_max": round(v[-1], 3),
                      "tflops": round(flops / (med * 1e-3) / 1e12, 1)}
        print(json.dumps(res))


if __name__ == "__main__":
    main()
