"""FLAME's vertex model on the GPU (gms_flame_lbs_forward / _backward through gms_b200.flame.NativeFlame) against the
float64 restatement of smplx.lbs (tests/flame_lbs_oracle): vertices and every gradient no further from float64 than the same
op sequence in fp32 ATen, within a factor of 4; bit-identical repeated backwards; FlameTrainer with a NativeFlame driver
against the ATen driver; sync-free steps; re-posing a reference-format checkpoint."""
import os

import numpy as np
import pytest
import torch

import flame_driver
import flame_lbs_oracle as oracle
from gms_b200 import _lib, io_ply, scenes
from gms_b200.flame import NativeFlame
from gms_b200.model import FlameGaussianModel, flame_transform_vertices
from gms_b200.trainer import FlameTrainer

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _synthetic_buffers(drv):
    return dict(v_template=drv.v_template, shapedirs=drv.shapedirs, posedirs=drv.posedirs, J_regressor=drv.J_regressor,
                parents=flame_driver.PARENTS, lbs_weights=drv.lbs_weights, faces=drv.faces)


def _flame_sized(V, seed, S=400):
    rs = np.random.RandomState(seed)
    v = rs.randn(V, 3) * 0.1
    jr = rs.rand(5, V) ** 8
    w = np.exp(-4 * ((v[:, None, :] / 0.1 - rs.randn(1, 5, 3) * 0.5) ** 2).sum(-1))
    t = lambda a: torch.tensor(a, dtype=torch.float32)
    return dict(v_template=t(v), shapedirs=t(rs.randn(V, 3, S) * 1e-3), posedirs=t(rs.randn(36, 3 * V) * 1e-3),
                J_regressor=t(jr / jr.sum(1, keepdims=True)), parents=(-1, 0, 1, 1, 1), lbs_weights=t(w / w.sum(1, keepdims=True)))


CASES = {
    "synthetic": lambda: (_synthetic_buffers(flame_driver.SyntheticFlame()), 100, 50),
    "flame V=5023 100/50": lambda: (_flame_sized(5023, 1), 100, 50),
    "flame V=5023 300/100": lambda: (_flame_sized(5023, 2), 300, 100),
    "V=33": lambda: (_flame_sized(33, 3), 100, 50),
}


def _params(V, n_shape, n_exp, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    enl = 8.35 * (1 + 0.3 * r(V, 3))
    enl[:7] = 0.0                      # zero and negative enlargement
    enl[7:14] = -enl[7:14].abs()
    return dict(shape=3.0 * r(1, n_shape), expression=3.0 * r(1, n_exp), pose=0.6 * r(1, 6), neck=0.6 * r(1, 3),
                transl=0.05 * r(1, 3), enl=enl, up=r(V, 3))


def _reference(buf, n_shape, n_exp, p, dtype, device):
    b = {k: (torch.as_tensor(v).to(device, dtype) if k not in ("parents", "faces") else v) for k, v in buf.items()}
    b["shapedirs"] = oracle.packed(b["shapedirs"], n_shape, n_exp)
    x = {k: p[k].to(device, dtype).requires_grad_(True) for k in ("shape", "expression", "pose", "neck", "transl", "enl")}
    out = oracle.transform(oracle.lbs(b, x["shape"], x["expression"], x["pose"], x["neck"], x["transl"]), x["enl"])
    (out * p["up"].to(device, dtype)).sum().backward()
    return out.detach().double().cpu(), {k: x[k].grad.double().cpu() for k in x}


def _native(fl, p):
    d = lambda t: t.float().contiguous().cuda()
    x = {k: d(p[k]) for k in ("shape", "expression", "pose", "neck", "transl", "enl")}
    ws = fl.workspace()
    out = torch.empty(fl.V, 3, device="cuda")
    vgrad = torch.full((fl.V, 3), float("nan"), device="cuda")
    a = fl._args(x["shape"], x["expression"], x["pose"], x["neck"], x["transl"], x["enl"], ws, vertices=out, vertices_grad=vgrad,
                 grads=[torch.full_like(x[k], float("nan")) for k in ("shape", "expression", "pose", "neck", "transl", "enl")])
    fl._launch("gms_flame_lbs_forward", a)
    assert bool((vgrad == 0).all()), "the forward zeroes the vertex gradient"
    vgrad.copy_(d(p["up"]))
    grads = []
    for _ in range(2):
        g = {k: torch.full_like(x[k], float("nan")) for k in x}
        a.d_shape, a.d_expression, a.d_pose, a.d_neck_pose, a.d_transl, a.d_enlargement = (g[k].data_ptr() for k in x)
        fl._launch("gms_flame_lbs_backward", a)
        grads.append(g)
    torch.cuda.synchronize()
    return out.double().cpu(), grads


@pytest.mark.parametrize("case", list(CASES))
def test_lbs_vs_float64_and_aten(case):
    buf, n_shape, n_exp = CASES[case]()
    fl = NativeFlame(**{k: v for k, v in buf.items()}, n_shape=n_shape, n_exp=n_exp)
    p = _params(fl.V, n_shape, n_exp, seed=len(case))
    ref_v, ref_g = _reference(buf, n_shape, n_exp, p, torch.float64, "cpu")
    at_v, at_g = _reference(buf, n_shape, n_exp, p, torch.float32, "cuda")
    nv, (g1, g2) = _native(fl, p)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), f"{k}: two backward calls differ"
    pairs = [("vertices", nv, at_v, ref_v)] + [(f"d_{k}", g1[k].double().cpu().reshape(ref_g[k].shape), at_g[k], ref_g[k]) for k in g1]
    for name, got, aten, ref in pairs:
        assert torch.isfinite(got).all(), name
        e_n, e_a = float((got - ref).abs().max()), float((aten - ref).abs().max())
        floor = 8 * 2.0 ** -24 * float(ref.abs().max())
        print(f"[flame-lbs] {case} {name}: max|native - f64| {e_n:.3e}, max|ATen fp32 - f64| {e_a:.3e}")
        assert e_n <= 4 * e_a + floor, name


def test_autograd_driver_matches_the_trainer_path():
    """NativeFlame as a driver (autograd Function, raw FLAME vertices) against the oracle in float64."""
    buf, n_shape, n_exp = CASES["V=33"]()
    fl = NativeFlame(**buf, n_shape=n_shape, n_exp=n_exp)
    p = _params(fl.V, n_shape, n_exp, seed=9)
    x = {k: p[k].cuda().requires_grad_(True) for k in ("shape", "expression", "pose", "neck", "transl")}
    v, lm = fl(shape_params=x["shape"], expression_params=x["expression"], pose_params=x["pose"], neck_pose=x["neck"], transl=x["transl"])
    assert lm is None and tuple(v.shape) == (1, fl.V, 3)
    out = flame_transform_vertices(v, p["enl"].cuda())
    (out * p["up"].cuda()).sum().backward()
    ref_v, ref_g = _reference(buf, n_shape, n_exp, p, torch.float64, "cpu")
    assert float((out.detach().double().cpu() - ref_v).abs().max()) <= 1e-5 * float(ref_v.abs().max())
    for k in x:
        r = ref_g[k]
        assert float((x[k].grad.double().cpu() - r).abs().max()) <= 1e-4 * float(r.abs().max()) + 1e-7, k


def _scene(drv_factory, K=10, W=256, H=256):
    torch.manual_seed(0)
    drv = drv_factory()
    faces = torch.from_numpy(np.asarray(drv.faces, np.int64)).cuda()
    m = FlameGaussianModel.create(drv, faces, K=K, seed=3)
    m.active_sh_degree = 1
    cams = [scenes.look_at_camera((0.35 * np.cos(a), 0.1, 0.35 * np.sin(a)), (0, 0, 0), W, H).to("cuda")
            for a in np.linspace(0, 2 * np.pi, 4, endpoint=False)]
    g = torch.Generator(device="cuda").manual_seed(1)
    gts = [torch.rand(3, H, W, device="cuda", generator=g) for _ in cams]
    return m, cams, gts, torch.ones(3, device="cuda")


def _train(native, steps=3, sync_check=False):
    syn = lambda: flame_driver.SyntheticFlame(rings=23, segments=24).cuda()
    drv = (lambda: NativeFlame(**_synthetic_buffers(syn()))) if native else syn
    m, cams, gts, bg = _scene(drv)
    t = FlameTrainer(m, bg)
    losses, launches = [], []
    for i in range(steps):
        _lib.launch_count(reset=True)
        if sync_check and i > 0:
            torch.cuda.set_sync_debug_mode("error")
        try:
            ln = t.step(cams[i % 4], gts[i % 4])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        launches.append(_lib.launch_count())
        losses.append(float(ln))
    return m, losses, launches


def test_trainer_with_native_flame_tracks_the_aten_driver():
    """Same buffers, same start.  First-step losses agree (the vertices differ only by rounding); after three steps every
    FLAME and Gaussian parameter is within DESIGN 4.2's bound: max(10x the native run-to-run difference, 1 % of its lr)."""
    m_n, l_n, launches = _train(True, sync_check=True)
    m_n2, _, _ = _train(True)
    m_a, l_a, launches_a = _train(False)
    print(f"[flame-lbs] losses native {l_n} ATen driver {l_a}; library launches per step native {launches} ATen {launches_a}")
    assert abs(l_n[0] - l_a[0]) <= 1e-5 * abs(l_a[0])
    assert launches[1:] == [launches_a[1] + 6] * 2
    from gms_b200.trainer import FlameOptimizationParams, flame_model_groups
    lrs = {g["name"]: g.get("lr", g.get("lr0")) for g in flame_model_groups(m_n, FlameOptimizationParams())}
    names = dict(_flame_shape="shape", _flame_exp="expression", _flame_pose="pose", _flame_neck_pose="neck_pose", _flame_trans="transl",
                 _vertices_enlargement="vertices_enlargement", _alpha="alpha", _opacity="opacity", _scales="scaling", _features="features")
    for n, g in names.items():
        p, p2, r = getattr(m_n, n).detach(), getattr(m_n2, n).detach(), getattr(m_a, n).detach()
        d, noise = float((p - r).abs().max()), float((p - p2).abs().max())
        bound = max(10 * noise, 1e-2 * lrs[g])
        over = int(((p - r).abs() > bound).sum())
        # Both drivers are deterministic, so the run-to-run term is 0 for the enlargement.  Its gradient is dL/dvertex times
        # the raw coordinate; where it is at rounding level it can take either sign once the two drivers' vertices differ
        # by one rounding (the likely cause; not traced element by element).  Adam (eps 1e-15) moves such an
        # element by +/- lr per step whatever its size: up to 2 % of the elements may take opposite steps (0.9 % measured),
        # and none may move further than three steps can (6 lr).
        allowed = 0.02 * p.numel() if n == "_vertices_enlargement" else max(2, 1e-4 * p.numel())
        print(f"[flame-lbs] after 3 steps {n}: max|native LBS - ATen driver| {d:.3e}, run-to-run {noise:.3e}, bound {bound:.3e}, {over} over")
        assert over <= allowed and d <= 6 * lrs[g], n


def test_reposed_checkpoint_renders_as_the_aten_driver(tmp_path):
    """A reference-format checkpoint whose point_cloud is to_point_cloud(): re-posed by from_checkpoint with an --animated
    style expression, drawn by FlameRenderer, against the same pose from the ATen driver."""
    from gms_b200.model import FlameCheckpoint
    from gms_b200.render import FlameRenderer
    syn = flame_driver.SyntheticFlame(rings=23, segments=24).cuda()
    m, cams, gts, bg = _scene(lambda: syn)
    t = FlameTrainer(m, bg)
    for i in range(2):
        t.step(cams[i], gts[i])
    fl = NativeFlame(**_synthetic_buffers(syn))
    ply = str(tmp_path / "point_cloud.ply")
    io_ply.save_flame_model(ply, m, point_cloud=fl.to_point_cloud())
    ck = FlameCheckpoint.load(ply, active_sh_degree=1)
    native = NativeFlame.from_checkpoint(io_ply.load_flame_model(ply)["point_cloud"])
    expr = torch.zeros(1, 50, device="cuda")
    expr[0, :5] = torch.tensor([1.5, -1.0, 0.5, 2.0, -0.5])
    v_n = ck.driver_vertices(native, expression_params=expr)
    v_a = ck.driver_vertices(syn, expression_params=expr)
    assert float((v_n - v_a).abs().max()) <= 1e-5 * float(v_a.abs().max())
    r = FlameRenderer(ck, 256, 256)
    img_n = r.render(cams[0], bg, vertices=v_n)[0].clone()
    img_a = r.render(cams[0], bg, vertices=v_a)[0].clone()
    d = float((img_n - img_a).abs().max())
    print(f"[flame-lbs] animated render: max|native pose - ATen pose| {d:.3e}")
    assert d <= 1e-3
