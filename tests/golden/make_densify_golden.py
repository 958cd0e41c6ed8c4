"""Generate densify.npz by running the reference's own GaussianModel (gs) and FlatGaussianModel (gs_flat) densification on
the CPU.

    python tests/golden/make_densify_golden.py        (needs /root/reference)

- `.cuda()` returns the tensor itself and device="cuda" allocations go to the CPU, as the other generators map them.
- torch.normal is wrapped: it draws z = torch.randn(std.shape), records z and returns z * std + mean.
- Per kind (gs, gs_flat) and max_screen_size (None, 20), one model of P = 96 rows built so that every class occurs: cloned,
  split, transparent, too large, split with too-large children, never visible (denom = 0).  Its statistics come from
  add_densification_stats over four synthetic frames; one torch.optim.Adam step (training_setup's groups) makes the moments
  non-zero; then densify_and_prune(0.0002, 0.005, extent, max_screen_size).  The state before and after is stored.
- reset_opacity of the gs_flat model, and the Adam state after a lone reset: a step with every gradient set whose opacity
  parameter was replaced (skipped), then a step with every gradient set.
- get_expon_lr_func (the xyz schedule of training_setup) at several iterations, and getNerfppNorm of five cameras.
- Every row's gradient norm, max scale and opacity is asserted to sit at least 1e-4 relative from its threshold, so the
  masks do not depend on the last bit of an exp or a sigmoid.
"""
import os
import sys
import types
from collections import namedtuple

import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)


def _stub(name, **attrs):
    m = types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


_stub("plyfile", PlyData=object, PlyElement=object)
_stub("simple_knn")
_stub("simple_knn._C", distCUDA2=None)
_stub("trimesh")
_stub("smplx")
_stub("smplx.lbs", lbs=None, batch_rodrigues=None, vertices2landmarks=None, find_dynamic_lmk_idx_and_bcoords=None)
_stub("smplx.utils", Struct=object, to_tensor=None, to_np=None, rot_mat_to_euler=None)
_stub("diff_gaussian_rasterization", GaussianRasterizationSettings=object, GaussianRasterizer=object)


def _cpu(fn):
    def f(*a, **k):
        if k.get("device", None) in ("cuda", torch.device("cuda")):
            k["device"] = "cpu"
        return fn(*a, **k)
    return f


for _n in ("zeros", "ones", "empty", "tensor", "full"):
    setattr(torch, _n, _cpu(getattr(torch, _n)))
torch.Tensor.cuda = lambda self, *a, **k: self
DRAWS = []
_randn = torch.randn


def _normal(*a, mean=None, std=None, **k):
    z = _randn(std.shape, dtype=std.dtype)
    DRAWS.append(z.clone())
    return z * std + mean


torch.normal = _normal

from scene.gaussian_model import GaussianModel  # noqa: E402
from games.flat_splatting.scene.flat_gaussian_model import FlatGaussianModel  # noqa: E402
from scene.dataset_readers import getNerfppNorm  # noqa: E402

P, EXTENT = 96, 4.0
Opt = namedtuple("Opt", "percent_dense position_lr_init position_lr_final position_lr_delay_mult position_lr_max_steps feature_lr "
                        "opacity_lr scaling_lr rotation_lr")
OPT = Opt(0.01, 0.00016, 0.0000016, 0.01, 30000, 0.0025, 0.05, 0.005, 0.001)


def make_model(kind, seed):
    g = torch.Generator().manual_seed(seed)
    cls = GaussianModel if kind == "gs" else FlatGaussianModel
    m = cls(3)
    cols = 3 if kind == "gs" else 2
    # row classes by index % 8: 0,1 small (clone if hot), 2,3 medium (split if hot), 4 large (> 0.1 extent), 5 medium with
    # children above 0.1 extent after / 1.6 only when > 0.64, 6 transparent, 7 never visible
    cls_ = torch.arange(P) % 8
    base = torch.tensor([0.01, 0.02, 0.1, 0.2, 0.8, 0.3, 0.05, 0.02])[cls_]
    scal = torch.log(base[:, None] * torch.exp(0.1 * torch.randn(P, cols, generator=g)))
    scal[cls_ == 5, 0] = np.log(0.9)        # a child above 0.4 = 0.1 extent: 0.9 / 1.6 = 0.56
    op = torch.randn(P, 1, generator=g)
    op[cls_ == 6] = -7.0 + 0.1 * torch.randn(int((cls_ == 6).sum()), 1, generator=g)
    feats = 0.3 * torch.randn(P, 16, 3, generator=g)
    m._xyz = torch.nn.Parameter(torch.randn(P, 3, generator=g))
    m._features_dc = torch.nn.Parameter(feats[:, :1].contiguous())
    m._features_rest = torch.nn.Parameter(feats[:, 1:].contiguous())
    m._scaling = torch.nn.Parameter(scal)
    m._rotation = torch.nn.Parameter(torch.randn(P, 4, generator=g))
    m._opacity = torch.nn.Parameter(op)
    m.max_radii2D = torch.zeros(P)
    m.spatial_lr_scale = EXTENT
    m.training_setup(OPT)
    # statistics over four frames: rows of class 7 never visible; hot rows (even index // 8) get a large gradient
    hot = (torch.arange(P) // 8) % 2 == 0
    for f in range(4):
        vs = types.SimpleNamespace(grad=torch.randn(P, 3, generator=g) * torch.where(hot, 6e-4, 2e-5)[:, None])
        vis = (cls_ != 7) & (torch.rand(P, generator=g) < 0.8)
        vis[0] = True
        m.add_densification_stats(vs, vis)
    # one Adam step so that the moments are non-zero
    for p in (m._xyz, m._features_dc, m._features_rest, m._opacity, m._scaling, m._rotation):
        p.grad = 1e-3 * torch.randn(p.shape, generator=g)
    m.optimizer.step()
    m.optimizer.zero_grad(set_to_none=True)
    return m


def state(m):
    out = dict(xyz=m._xyz, scaling=m._scaling, rotation=m._rotation, opacity=m._opacity,
               features=torch.cat([m._features_dc, m._features_rest], dim=1))
    st = {g["name"]: m.optimizer.state[g["params"][0]] for g in m.optimizer.param_groups}
    for n, k in (("xyz", "xyz"), ("scaling", "scaling"), ("rotation", "rotation"), ("opacity", "opacity")):
        out["m_" + n], out["v_" + n] = st[k]["exp_avg"], st[k]["exp_avg_sq"]
    out["m_features"] = torch.cat([st["f_dc"]["exp_avg"], st["f_rest"]["exp_avg"]], dim=1)
    out["v_features"] = torch.cat([st["f_dc"]["exp_avg_sq"], st["f_rest"]["exp_avg_sq"]], dim=1)
    return {k: v.detach().clone().numpy() for k, v in out.items()}


def check_margins(m, extent, size):
    g = (m.xyz_gradient_accum / m.denom).squeeze(1)
    g[g.isnan()] = 0
    smax = m.get_scaling.max(dim=1).values
    rel = lambda a, t: ((a - t).abs() / t).min()
    assert rel(g[g > 0], 0.0002) > 1e-4
    assert rel(smax, 0.01 * extent) > 1e-4 and rel(smax, 0.1 * extent) > 1e-4 and rel(smax / 1.6, 0.1 * extent) > 1e-4
    assert rel(m.get_opacity.squeeze(1), 0.005) > 1e-4


def main():
    out = {}
    for kind in ("gs", "gs_flat"):
        for mss in (None, 20):
            tag = f"{kind}_{'none' if mss is None else mss}_"
            m = make_model(kind, seed=7 if kind == "gs" else 8)
            check_margins(m, EXTENT, mss)
            before = state(m)
            for k, v in before.items():
                out[tag + "in_" + k] = v
            out[tag + "accum"] = m.xyz_gradient_accum.squeeze(1).numpy().copy()
            out[tag + "denom"] = m.denom.squeeze(1).numpy().copy()
            g = (m.xyz_gradient_accum / m.denom)
            g[g.isnan()] = 0.0
            smax = m.get_scaling.max(dim=1).values
            split_mask = (g.squeeze(1) >= 0.0002) & (smax > 0.01 * EXTENT)
            DRAWS.clear()
            m.densify_and_prune(0.0002, 0.005, EXTENT, mss)
            z = DRAWS[0]
            S = int(split_mask.sum())
            normals = torch.zeros(P, 2, 3)
            normals[split_mask, 0] = z[:S]
            normals[split_mask, 1] = z[S:]
            out[tag + "normals"] = normals.numpy()
            for k, v in state(m).items():
                out[tag + "out_" + k] = v
            out[tag + "out_accum"] = m.xyz_gradient_accum.squeeze(1).numpy().copy()
    # reset_opacity and a lone reset's Adam state (gs_flat)
    m = make_model("gs_flat", seed=9)
    g = torch.Generator().manual_seed(10)
    params = lambda: [m._xyz, m._features_dc, m._features_rest, m._opacity, m._scaling, m._rotation]
    grads_a = [1e-3 * torch.randn(p.shape, generator=g) for p in params()]
    grads_b = [1e-3 * torch.randn(p.shape, generator=g) for p in params()]
    for k, v in state(m).items():
        out["reset_in_" + k] = v
    for p, gr in zip(params(), grads_a):
        p.grad = gr.clone()
    m.reset_opacity()
    for k, v in state(m).items():
        out["reset_mid_" + k] = v
    m.optimizer.step()
    m.optimizer.zero_grad(set_to_none=True)
    for p, gr in zip(params(), grads_b):
        p.grad = gr.clone()
    m.optimizer.step()
    for k, v in state(m).items():
        out["reset_out_" + k] = v
    for i, n in enumerate(("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")):
        out["reset_grad_a_" + n], out["reset_grad_b_" + n] = grads_a[i].numpy(), grads_b[i].numpy()
    out["reset_steps"] = np.array([int(m.optimizer.state[gr["params"][0]]["step"]) for gr in m.optimizer.param_groups])
    # the xyz learning-rate schedule and the scene extent
    its = np.array([0, 1, 100, 500, 1000, 7000, 15000, 29999, 30000, 40000])
    out["lr_iters"], out["lr_xyz"] = its, np.array([m.xyz_scheduler_args(int(i)) for i in its])
    Cam = namedtuple("Cam", "R T")
    rng = np.random.default_rng(11)
    cams = []
    for _ in range(5):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        w, x, y, zq = q
        R = np.array([[1 - 2 * (y * y + zq * zq), 2 * (x * y - w * zq), 2 * (x * zq + w * y)],
                      [2 * (x * y + w * zq), 1 - 2 * (x * x + zq * zq), 2 * (y * zq - w * x)],
                      [2 * (x * zq - w * y), 2 * (y * zq + w * x), 1 - 2 * (x * x + y * y)]])
        cams.append(Cam(R, rng.normal(size=3) * 3))
    norm = getNerfppNorm(cams)
    out["cam_R"] = np.stack([c.R for c in cams])
    out["cam_T"] = np.stack([c.T for c in cams])
    out["cam_radius"] = np.array(norm["radius"])
    np.savez_compressed(os.path.join(HERE, "densify.npz"), **out)
    print({k: v.shape for k, v in out.items() if k.endswith("out_xyz")})


if __name__ == "__main__":
    main()
