"""Training-step and densification timings of free flat Gaussians (train.py --gs_type gs_flat).

    python tools/free_train_eval.py --bench [--runs 5] [--steps 50] > free_train_eval.txt
    python tools/free_train_eval.py                 # the same arms on a small scene (a quick end-to-end run)

Workload (--bench): 1M gs_flat Gaussians (scenes.flat_gaussians, as raw parameters), 1080p, 16 ring cameras, a fixed random
ground truth per camera, white background.  Arms, alternated `--runs` times, CUDA events over `--steps` steps after a warm-up
of one step per camera, in a window without densification (the densification statistics are gathered every step):
  native      FreeTrainer: one gms_free_train_frame per step with the statistics fused, the SH Adam step fused into the
              frame, FlatAdam for the rest;
  autograd    the reference's step shape on the library's kernels: getters in ATen, the autograd shim rasterizer, the fused
              loss, add_densification_stats in ATen, torch.optim.Adam (eps 1e-15) over the reference's six groups.
Then one densify_and_prune per arm at that size, on the statistics it gathered (host clock around work that ends in a
device synchronisation): native = gms_densify_plan + gms_densify_apply + FlatAdam.resize; autograd = the ATen restatement
(tests/densify_oracle.py) with the parameters and the torch.optim.Adam state rebuilt as the reference's cat / mask does.
Reported: ms per step, library launches per step, each arm's first-step loss from the same parameters, ms per densification
and the new P.  The card's name, power limit and SM clock are read in the same run (nvidia-smi, read-only query)."""
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
from torch import nn  # noqa: E402

import densify_oracle as D  # noqa: E402
from gms_b200 import _lib, scenes  # noqa: E402
from gms_b200.losses import fused_training_loss  # noqa: E402
from gms_b200.model import FreeGaussianModel  # noqa: E402
from gms_b200.trainer import FreeOptimizationParams, FreeTrainer, expon_lr  # noqa: E402

NO_DENSIFY = dict(densify_from_iter=10 ** 9, densify_until_iter=10 ** 9, opacity_reset_interval=10 ** 9, iterations=10 ** 9)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable: {e}"


def raw_flat(P, seed=0):
    g = scenes.flat_gaussians(P, seed)
    return dict(xyz=g["means3D"], scaling=torch.log(g["scales"][:, 1:]).contiguous(), rotation=g["rotations"], features=g["shs"],
                opacity=torch.logit(g["opacities"]))


class AutogradStep:
    """GaussianModel's training iteration on the library's kernels through autograd (flat_gaussian_model.py getters,
    GaussianRasterizer, the fused L1 + SSIM loss, add_densification_stats, torch.optim.Adam)."""

    def __init__(self, raw, bg, extent, dev, opt=FreeOptimizationParams(**NO_DENSIFY)):
        P_ = lambda t: nn.Parameter(t.to(dev).float().contiguous())
        self.xyz, self.scaling, self.rotation, self.opacity = P_(raw["xyz"]), P_(raw["scaling"]), P_(raw["rotation"]), P_(raw["opacity"])
        self.dc, self.rest = P_(raw["features"][:, :1]), P_(raw["features"][:, 1:])
        self.o, self.extent, self.bg, self.it = opt, extent, bg, 0
        self._adam()
        self.accum = torch.zeros(self.xyz.shape[0], device=dev)
        self.denom = torch.zeros(self.xyz.shape[0], device=dev)

    def params(self):
        return dict(xyz=self.xyz, f_dc=self.dc, f_rest=self.rest, opacity=self.opacity, scaling=self.scaling, rotation=self.rotation)

    def _adam(self, state=None):
        o = self.o
        lrs = dict(xyz=expon_lr(self.it, o.position_lr_init * self.extent, o.position_lr_final * self.extent, 0, o.position_lr_delay_mult,
                                o.position_lr_max_steps), f_dc=o.feature_lr, f_rest=o.feature_lr / 20, opacity=o.opacity_lr,
                   scaling=o.scaling_lr, rotation=o.rotation_lr)
        self.adam = torch.optim.Adam([dict(params=[p], lr=lrs[n], name=n) for n, p in self.params().items()], lr=0.0, eps=1e-15)
        if state:
            for g in self.adam.param_groups:
                self.adam.state[g["params"][0]] = state[g["name"]]

    def step(self, cam, gt):
        import diff_gaussian_rasterization as dgr
        self.it += 1
        o = self.o
        self.adam.param_groups[0]["lr"] = expon_lr(self.it, o.position_lr_init * self.extent, o.position_lr_final * self.extent, 0,
                                                   o.position_lr_delay_mult, o.position_lr_max_steps)
        s = torch.exp(self.scaling)
        scales = torch.cat([torch.full((s.shape[0], 1), 1e-8, device=s.device), s], 1)
        m2d = torch.zeros_like(self.xyz, requires_grad=True)
        rs = dgr.GaussianRasterizationSettings(
            image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
            bg=self.bg, scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
            sh_degree=3, campos=cam.camera_center, prefiltered=False, debug=False, antialiasing=False)
        image, radii, _ = dgr.GaussianRasterizer(raster_settings=rs)(
            means3D=self.xyz, means2D=m2d, opacities=torch.sigmoid(self.opacity), shs=torch.cat((self.dc, self.rest), dim=1),
            scales=scales, rotations=torch.nn.functional.normalize(self.rotation))
        loss = fused_training_loss(image, gt, o.lambda_dssim)
        loss.backward()
        with torch.no_grad():
            vis = radii > 0
            self.accum[vis] += torch.norm(m2d.grad[vis, :2], dim=-1)
            self.denom[vis] += 1
        self.adam.step()
        self.adam.zero_grad(set_to_none=True)
        return loss.detach()

    def densify(self, size_prune=False):
        """densify_and_prune through the ATen restatement; parameters and Adam state rebuilt at the new size."""
        st = {g["name"]: self.adam.state[g["params"][0]] for g in self.adam.param_groups}
        state = dict(xyz=self.xyz.data, scaling=self.scaling.data, rotation=self.rotation.data, opacity=self.opacity.data,
                     features=torch.cat([self.dc.data, self.rest.data], 1))
        for n, k in (("xyz", "xyz"), ("scaling", "scaling"), ("rotation", "rotation"), ("opacity", "opacity")):
            state["m_" + n], state["v_" + n] = st[k]["exp_avg"], st[k]["exp_avg_sq"]
        state["m_features"] = torch.cat([st["f_dc"]["exp_avg"], st["f_rest"]["exp_avg"]], 1)
        state["v_features"] = torch.cat([st["f_dc"]["exp_avg_sq"], st["f_rest"]["exp_avg_sq"]], 1)
        normals = torch.randn(self.xyz.shape[0], 2, 3, device=self.xyz.device)
        out, _, counts = D.densify(state, self.accum, self.denom, normals, self.extent, size_prune=size_prune)
        self.xyz, self.scaling, self.rotation, self.opacity = (nn.Parameter(out[n]) for n in ("xyz", "scaling", "rotation", "opacity"))
        self.dc, self.rest = nn.Parameter(out["features"][:, :1].contiguous()), nn.Parameter(out["features"][:, 1:].contiguous())
        new = {}
        for n, k, sl in (("xyz", "xyz", None), ("scaling", "scaling", None), ("rotation", "rotation", None), ("opacity", "opacity", None),
                         ("features", "f_dc", slice(0, 1)), ("features", "f_rest", slice(1, None))):
            m, v = out["m_" + n], out["v_" + n]
            if sl is not None:
                m, v = m[:, sl].contiguous(), v[:, sl].contiguous()
            new[k] = dict(step=st[k]["step"], exp_avg=m, exp_avg_sq=v)
        self._adam(new)
        self.accum = torch.zeros(self.xyz.shape[0], device=self.xyz.device)
        self.denom = torch.zeros_like(self.accum)
        return counts


def time_arms(arms, cams, gts, runs, steps):
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
        print(f"  {name:10s} ms/step {np.mean(ms):8.3f} (runs {', '.join(f'{m:.3f}' for m in ms)}), "
              f"launches/step {rs[-1][1]:.1f}, first-step loss {first[name]:.7f}")
    return res


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench", action="store_true", help="the full workload (1M gs_flat Gaussians, 1080p, 16 cameras)")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("free_train_eval.py times GPU steps: no CUDA device")
    P, W, H, ncam = (1_000_000, 1920, 1080, 16) if args.bench else (50_000, 480, 270, 4)
    dev = "cuda"
    print(card())
    cams = [c.to(dev) for c in scenes.ring_cameras(ncam // 2, 3.4, W, H, elevation_deg=15.0) +
            scenes.ring_cameras(ncam - ncam // 2, 4.4, W, H, elevation_deg=38.0, phase=0.3)]
    for i, c in enumerate(cams):
        c.uid = i
    g = torch.Generator(device=dev).manual_seed(0)
    gts = [torch.rand(3, H, W, generator=g, device=dev) for _ in cams]
    bg = torch.ones(3, device=dev)
    extent = scenes.camera_extent(cams)
    raw = raw_flat(P)
    print(f"== gs_flat: P = {P}, {W}x{H}, {len(cams)} cameras, extent {extent:.3f}, {args.runs} alternating runs x {args.steps} steps")
    model = FreeGaussianModel(raw["xyz"], raw["scaling"], raw["rotation"], raw["features"], raw["opacity"], "gs_flat", dev, 3)
    native = FreeTrainer(model, bg, extent, FreeOptimizationParams(**NO_DENSIFY))
    auto = AutogradStep(raw, bg, extent, dev)
    time_arms({"native": native.step, "autograd": auto.step}, cams, gts, args.runs, args.steps)
    print(f"  native overflows {native.frame.overflows}")
    for name, fn in (("native", lambda: native.densify(size_prune=False)), ("autograd", lambda: auto.densify(size_prune=False))):
        ms, counts = timed(fn)
        print(f"  {name:10s} densify_and_prune at P = {P}: {ms:8.3f} ms -> new P {counts[0]} "
              f"(kept {counts[1]}, clones {counts[2]}, split pairs {counts[3]}, pruned {counts[4]})")
    print(card())


if __name__ == "__main__":
    main()
