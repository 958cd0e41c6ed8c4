"""Training-step timings of a gs_multi_mesh scene with a different splat count per mesh (train.py --gs_type gs_multi_mesh
--num_splats 2 4 5 9).

    python tools/multi_mesh_eval.py --bench [--runs 5] [--steps 50] > multi_mesh_eval.txt
    python tools/multi_mesh_eval.py                 # the same arms on a small scene (a quick end-to-end run)

Workload (--bench): four disjoint 100k-face objects (scenes.object_mesh, laid out as bench.py's gs_multi_mesh scene),
K = (2, 4, 5, 9) splats per face, so P = 2.0M; 1080p, 16 ring cameras, a fixed random ground truth per camera.
Arms, alternated `--runs` times, CUDA events over `--steps` steps after a warm-up of one step per camera:
  native      MeshTrainer(native=True) on the segmented model: one gms_train_frame per step (the expansion launched once
              per mesh), the SH Adam step fused into the frame, FlatAdam for the rest;
  autograd    MeshTrainer(fast=True, native=False) on the same model: expand_fused (per mesh, then cat), the autograd shim
              rasterizer, the fused loss, FlatAdam;
  reference   the reference's step shape: expand_per_mesh, the shim rasterizer, the ATen loss (tests/aten_reference.py),
              torch.optim.Adam over per-mesh parameter lists (gaussian_multi_mesh_model.py:201-216);
and, for what the per-mesh launches cost, K = (5, 5, 5, 5) (P = 2.0M) natively as four segments against the merged
single-segment model.  Reported: ms per step, library launches per step, and each arm's first-step loss from the same
parameters.  The card's name, power limit and SM clock are read in the same run (nvidia-smi, read-only query)."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import aten_reference  # noqa: E402
from gms_b200 import _lib, scenes  # noqa: E402
from gms_b200.model import MultiMeshGaussianModel  # noqa: E402
from gms_b200.optim import REFERENCE_LRS  # noqa: E402
from gms_b200.trainer import MeshTrainer  # noqa: E402

CENTRES = [(-0.75, -0.75, 0.0), (0.75, -0.75, 0.0), (-0.75, 0.75, 0.0), (0.75, 0.75, 0.0)]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable: {e}"


def meshes(F_each, Ks, seed=0):
    plist = []
    for k, (c, K) in enumerate(zip(CENTRES, Ks)):
        v, f = scenes.object_mesh(F_each)
        plist.append(scenes.init_mesh_gaussians(v * 0.55 + np.float32(c), f, K, seed=seed + k, trained_like=True))
    return plist


class ReferenceStep:
    """The reference's training step shape on per-mesh parameter lists: expand_per_mesh -> getters -> GaussianRasterizer
    -> ATen L1 + SSIM -> backward -> torch.optim.Adam (eps 1e-15) -> zero_grad."""

    def __init__(self, plist, bg, dev, lam=0.2):
        import torch.nn as nn
        P = lambda t: nn.Parameter(t.to(dev).float().contiguous())
        self.v = [P(p.vertices) for p in plist]
        self.f = [p.faces.to(dev) for p in plist]
        self.a = [P(p._alpha) for p in plist]
        self.s = [P(p._scale) for p in plist]
        self.dc = P(torch.cat([p._features_dc for p in plist]))
        self.rest = P(torch.cat([p._features_rest for p in plist]))
        self.op = P(torch.cat([p._opacity for p in plist]))
        lr = REFERENCE_LRS
        self.opt = torch.optim.Adam([{"params": self.a, "lr": lr["alpha"]}, {"params": self.v, "lr": lr["vertices"]},
                                     {"params": [self.dc], "lr": lr["f_dc"]}, {"params": [self.rest], "lr": lr["f_rest"]},
                                     {"params": [self.op], "lr": lr["opacity"]}, {"params": self.s, "lr": lr["scaling"]}],
                                    lr=0.0, eps=1e-15)
        self.bg, self.lam = bg, lam

    def step(self, cam, gt):
        import diff_gaussian_rasterization as dgr
        xyz, sl, rr = MultiMeshGaussianModel.expand_per_mesh(self.v, self.f, self.a, self.s)
        rs = dgr.GaussianRasterizationSettings(
            image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
            bg=self.bg, scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
            sh_degree=3, campos=cam.camera_center, prefiltered=False, debug=False, antialiasing=False)
        image, _, _ = dgr.GaussianRasterizer(raster_settings=rs)(
            means3D=xyz, means2D=torch.zeros_like(xyz, requires_grad=True), opacities=torch.sigmoid(self.op),
            shs=torch.cat((self.dc, self.rest), dim=1), scales=torch.exp(sl), rotations=torch.nn.functional.normalize(rr))
        loss = aten_reference.training_loss(image, gt, self.lam)
        loss.backward()
        self.opt.step()
        self.opt.zero_grad(set_to_none=False)
        return loss.detach()


def time_arms(arms, cams, gts, runs, steps):
    """arms: name -> step(cam, gt).  Warm-up of one step per camera, then `runs` alternating runs of `steps` steps each."""
    first = {}
    for name, step in arms.items():
        first[name] = float(step(cams[0], gts[0]))
        for i in range(1, len(cams)):
            step(cams[i], gts[i])
    torch.cuda.synchronize()
    res = {name: [] for name in arms}
    for run in range(runs):
        for name, step in arms.items():
            _lib.launch_count(reset=True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(steps):
                j = (run * steps + i) % len(cams)
                step(cams[j], gts[j])
            e1.record()
            torch.cuda.synchronize()
            res[name].append((e0.elapsed_time(e1) / steps, _lib.launch_count(reset=True) / steps))
    for name, rs in res.items():
        ms = [r[0] for r in rs]
        print(f"  {name:22s} ms/step {np.mean(ms):8.3f} (runs {', '.join(f'{m:.3f}' for m in ms)}), "
              f"launches/step {rs[-1][1]:.1f}, first-step loss {first[name]:.7f}")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench", action="store_true", help="the full workload (4 x 100k faces, K = (2, 4, 5, 9), 1080p, 16 cameras)")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_mesh_eval.py times GPU steps: no CUDA device")
    F_each, W, H, ncam = (100_000, 1920, 1080, 16) if args.bench else (5_000, 480, 270, 4)
    dev = "cuda"
    print(card())
    cams = [c.to(dev) for c in scenes.ring_cameras(ncam // 2, 3.4, W, H, elevation_deg=15.0) +
            scenes.ring_cameras(ncam - ncam // 2, 4.4, W, H, elevation_deg=38.0, phase=0.3)]
    g = torch.Generator(device=dev).manual_seed(0)
    gts = [torch.rand(3, H, W, generator=g, device=dev) for _ in cams]
    bg = torch.ones(3, device=dev)

    Ks = (2, 4, 5, 9)
    plist = meshes(F_each, Ks)
    F = sum(p.faces.shape[0] for p in plist)
    P = sum(p._scale.shape[0] for p in plist)
    print(f"== K = {Ks}: F = {F}, P = {P}, {W}x{H}, {len(cams)} cameras, {args.runs} alternating runs x {args.steps} steps")
    native = MeshTrainer(MultiMeshGaussianModel.from_mesh_params(plist, dev, packed_features=True), bg, native=True)
    autograd = MeshTrainer(MultiMeshGaussianModel.from_mesh_params(plist, dev, packed_features=True), bg, native=False)
    ref = ReferenceStep(plist, bg, dev)
    time_arms({"native": native.step, "autograd": autograd.step, "reference": ref.step}, cams, gts, args.runs, args.steps)
    print(f"  native overflows {native._frame.overflows}")
    del native, autograd, ref
    torch.cuda.empty_cache()

    plist = meshes(F_each, (5, 5, 5, 5))
    P = sum(p._scale.shape[0] for p in plist)
    print(f"== K = (5, 5, 5, 5): P = {P}, native, four segments against the merged model")
    seg = MeshTrainer(MultiMeshGaussianModel.from_mesh_params(plist, dev, packed_features=True, segmented=True), bg, native=True)
    merged = MeshTrainer(MultiMeshGaussianModel.from_mesh_params(plist, dev, packed_features=True), bg, native=True)
    assert seg.model.segments is not None and merged.model.segments is None
    time_arms({"native, 4 segments": seg.step, "native, merged": merged.step}, cams, gts, args.runs, args.steps)
    print(f"  overflows: segmented {seg._frame.overflows}, merged {merged._frame.overflows}")
    print(card())


if __name__ == "__main__":
    main()
