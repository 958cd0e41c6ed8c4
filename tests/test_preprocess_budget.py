"""The preprocess backward per element: every parameter gradient against the float64 reference of oracle/preprocess64.py,
within its a-priori error budget (the soundness argument heads that module).

The global stage-2 measure (max |gpu - oracle| / max |oracle|, DESIGN.md 2.2) cannot see a Gaussian whose gradient is small
next to the largest one.  These CPU tests show that
  * the reference computes the operation itself: float64 autograd of the forward maths agrees to 1e-10 per element,
  * every correct fp32 implementation lies inside the budget on every scene: the C oracle, the product's
    gms_preprocess.cuh compiled for the CPU (tests/hostshim), and a plain fp32 evaluation of the reference's own tree,
  * the budget has teeth: six plausible kernel bugs pass the old floor on some scene and fail the per-element check on
    every scene where they change the operation,
  * the budget is not vacuous (its median relative size is printed and bounded)."""
import ctypes as C

import numpy as np
import pytest
import torch

import preprocess_budget_cases as pbc
from gms_b200 import scenes
from helpers import random_gaussians, settings_from_camera
from hostshim import build_shim
from oracle import preprocess64, raster

# the old stage-2 floor (tests/gpu_helpers.py STAGE2_TOL, 5e-5 for the other gradients): max |err| / max |ref| per tensor
OLD_FLOOR = {"scales": 5e-3, "rotations": 5e-3, "cov3D_precomp": 5e-3, "means3D": 5e-4}
# outputs of raster.preprocess_backward compared per element (dL_dcov3D is written for every Gaussian by the oracle)
KEYS = {"means3D": "dL_dmeans3D", "opacities": "dL_dopacity", "shs": "dL_dsh", "colors_precomp": "dL_dcolors_precomp",
        "scales": "dL_dscales", "rotations": "dL_drotations", "cov3D": "dL_dcov3D"}


@pytest.fixture(scope="module")
def shim():
    return C.CDLL(build_shim.build())


@pytest.fixture(scope="module")
def cases():
    """name -> (st, record, reference); the record is the C oracle's composite backward under random upstream gradients."""
    out = {}
    for name, build in pbc.SCENES.items():
        S, g = build()
        st = pbc.forward(S, g)
        dg = pbc.record(st, *pbc.upstream(S))
        out[name] = (st, dg, preprocess64.preprocess_backward64(st, dg))
    return out


def _oracle(st, dg):
    fed = dict(dL_dmean2D=dg[:, 0:2], dL_dconic=dg[:, 2:5], dL_dopacity=dg[:, 5], dL_dcolor=dg[:, 6:9], dL_dinvdepth=dg[:, 9])
    o = raster.preprocess_backward(st, fed)
    return {k: o[v] for k, v in KEYS.items() if o.get(v) is not None}


def _shim(shim, st, dg):
    S, inp = st.settings, st.inputs
    P, M = st.radii.shape[0], st.cs.M
    f = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
    p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)
    view, proj, campos = f(np.reshape(S.viewmatrix, 16)), f(np.reshape(S.projmatrix, 16)), f(np.reshape(S.campos, 3))
    rec_ = [np.ascontiguousarray(dg[:, a:b], np.float32) for a, b in ((0, 2), (2, 5), (5, 6), (6, 9), (9, 10))]
    o = dict(means3D=np.zeros((P, 3), np.float32), cov3D=np.zeros((P, 6), np.float32), opacities=np.zeros(P, np.float32))
    if inp["shs"] is not None:
        o["shs"] = np.zeros((P, M, 3), np.float32)
    if inp["scales"] is not None:
        o["scales"], o["rotations"] = np.zeros((P, 3), np.float32), np.zeros((P, 4), np.float32)
    rc = shim.shim_preprocess_backward(P, S.sh_degree, M, S.image_width, S.image_height, C.c_float(S.tanfovx), C.c_float(S.tanfovy),
                                       C.c_float(S.scale_modifier), int(S.antialiasing), p(st.radii), p(inp["means3D"]),
                                       p(inp["scales"]), p(inp["rotations"]), p(inp["opacities"]), p(inp["shs"]), p(view), p(proj),
                                       p(campos), p(f(st.cov3Ds)), p(st.clamped), *map(p, rec_), p(o["means3D"]), p(o["cov3D"]),
                                       p(o.get("shs")), p(o.get("scales")), p(o.get("rotations")), p(o["opacities"]))
    assert rc == 0
    return o


def _f32(st, dg, bug=None):
    o = preprocess64.preprocess_backward_f32(st, dg, bug)
    return {k: o[v] for k, v in KEYS.items() if o.get(v) is not None}


def _within(got, r, vis):
    """got keyed like KEYS -> worst |got - ref64| / budget per key over the visible Gaussians (the C oracle also writes the
    covariance gradient of culled ones)."""
    out = {}
    for k, a in got.items():
        ratio = pbc.budget_ratios(a, r["ref64"][KEYS[k]], r["budget"][KEYS[k]])[vis]
        out[k] = float(np.nan_to_num(ratio, nan=np.inf).max()) if ratio.size else 0.0
    return out


def _floor(got, ref):
    """The old global measure per tensor: passes when max |err| / max |ref| stays under the stage-2 floor."""
    ok = True
    for k, a in got.items():
        kg = "cov3D_precomp" if k == "cov3D" else k
        b = np.asarray(ref[k], np.float64).reshape(np.shape(a))
        e = np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30) if b.size else 0.0
        ok &= e <= OLD_FLOOR.get(kg, 5e-5)
    return ok


# ------------------------------------------------------------------------------------------------ the formula, independently
def _sh_to_rgb(deg, sh, d):
    """utils/sh_utils.py:eval_sh with the fp32 values of the SH constants (those of the operation)."""
    C0, C1, C2, C3 = preprocess64.SH_C0, preprocess64.SH_C1, preprocess64.SH_C2, preprocess64.SH_C3
    x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    res = C0 * sh[:, 0]
    if deg > 0:
        res = res - C1 * y * sh[:, 1] + C1 * z * sh[:, 2] - C1 * x * sh[:, 3]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        res = (res + C2[0] * xy * sh[:, 4] + C2[1] * yz * sh[:, 5] + C2[2] * (2 * zz - xx - yy) * sh[:, 6]
               + C2[3] * xz * sh[:, 7] + C2[4] * (xx - yy) * sh[:, 8])
    if deg > 2:
        res = (res + C3[0] * y * (3 * xx - yy) * sh[:, 9] + C3[1] * xy * z * sh[:, 10]
               + C3[2] * y * (4 * zz - xx - yy) * sh[:, 11] + C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[:, 12]
               + C3[4] * x * (4 * zz - xx - yy) * sh[:, 13] + C3[5] * z * (xx - yy) * sh[:, 14]
               + C3[6] * x * (xx - 3 * yy) * sh[:, 15])
    return res


def _autograd(st, dg):
    """float64 autograd of the forward maths (oracle/torch_dense.py's restatement) on the visible Gaussians: the gradient of
    sum(record * forward outputs), with the conic xy weighted 2x (the record holds it in the upstream's half convention)."""
    from oracle.torch_dense import quat_to_R
    S, inp = st.settings, st.inputs
    vis = st.radii > 0
    dt = torch.float64
    t = lambda a: torch.tensor(np.asarray(a, np.float64)[vis], dtype=dt, requires_grad=True)
    m, sc, q, op = t(inp["means3D"]), t(inp["scales"]), t(inp["rotations"]), t(np.reshape(inp["opacities"], (-1, 1)))
    sh = t(inp["shs"])
    view = torch.tensor(np.asarray(S.viewmatrix, np.float64), dtype=dt).reshape(4, 4)
    proj = torch.tensor(np.asarray(S.projmatrix, np.float64), dtype=dt).reshape(4, 4)
    hom = torch.cat([m, torch.ones(m.shape[0], 1, dtype=dt)], 1)
    pv, ph = (hom @ view)[:, :3], hom @ proj
    pw = 1.0 / (ph[:, 3] + preprocess64.EPS_W)
    R = quat_to_R(q)
    Mx = R * (preprocess64.f32(S.scale_modifier) * sc)[:, None, :]
    Sig = Mx @ Mx.transpose(1, 2)
    Sig.retain_grad()
    fx = preprocess64.f32(np.float32(S.image_width) / (np.float32(2) * np.float32(S.tanfovx)))
    fy = preprocess64.f32(np.float32(S.image_height) / (np.float32(2) * np.float32(S.tanfovy)))
    tx, ty, tz = pv[:, 0], pv[:, 1], pv[:, 2]
    z0 = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, z0, -fx * tx / tz ** 2], 1), torch.stack([z0, fy / tz, -fy * ty / tz ** 2], 1)], 1)
    Wm = view[:3, :3].T
    T = J @ Wm
    cov2 = T @ Sig @ T.transpose(1, 2)
    a0, b, c0 = cov2[:, 0, 0], cov2[:, 0, 1], cov2[:, 1, 1]
    a, c = a0 + preprocess64.HVAR, c0 + preprocess64.HVAR
    det = a * c - b * b
    con = torch.stack([c / det, -b / det, a / det], 1)
    h = torch.sqrt((a0 * c0 - b * b) / det) if S.antialiasing else torch.ones_like(det)
    d = m - torch.tensor(np.asarray(S.campos, np.float64), dtype=dt)
    d = d / d.norm(dim=1, keepdim=True)
    rgb = torch.clamp(_sh_to_rgb(S.sh_degree, sh, d) + 0.5, min=0.0)
    g = torch.tensor(np.asarray(dg, np.float64)[vis], dtype=dt)
    loss = (g[:, 0] * ph[:, 0] * pw + g[:, 1] * ph[:, 1] * pw + g[:, 2] * con[:, 0] + 2 * g[:, 3] * con[:, 1] + g[:, 4] * con[:, 2]
            + g[:, 5] * op[:, 0] * h + (g[:, 6:9] * rgb).sum(1) + g[:, 9] / tz).sum()
    loss.backward()
    s6 = Sig.grad
    cov = torch.stack([s6[:, 0, 0], s6[:, 0, 1] + s6[:, 1, 0], s6[:, 0, 2] + s6[:, 2, 0], s6[:, 1, 1], s6[:, 1, 2] + s6[:, 2, 1],
                       s6[:, 2, 2]], 1)
    return dict(dL_dmeans3D=m.grad, dL_dscales=sc.grad, dL_drotations=q.grad, dL_dopacity=op.grad, dL_dsh=sh.grad,
                dL_dcov3D=cov), Sig.detach()


@pytest.mark.parametrize("aa", [False, True])
def test_reference_is_the_derivative_of_the_forward(aa):
    """Away from the guard band and with the det^2 + 1e-7 term switched off, the reference is the true derivative: float64
    autograd of the forward maths agrees per element to 1e-10 of the element (plus 1e-13 of the component's largest)."""
    S = settings_from_camera(scenes.look_at_camera((2.2, 1.5, 0.9), (0, 0, 0), 160, 112), antialiasing=aa)
    g = random_gaussians(200, seed=8, extent=0.6, scale_mu=-2.4, flat_frac=0.0)
    st = pbc.forward(S, g)
    dg = pbc.record(st, *pbc.upstream(S))
    vis = st.radii > 0
    auto, sig = _autograd(st, dg)
    st.cov3Ds = st.cov3Ds.astype(np.float64)          # the reference reads the forward's covariance: give it the float64 one
    iu = ([0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2])
    st.cov3Ds[vis] = sig.numpy()[:, iu[0], iu[1]]
    st.clamped = np.asarray(st.clamped).copy()
    r = preprocess64.preprocess_backward64(st, dg, det2_eps=0.0)
    assert vis.sum() > 100 and not r["ambiguous"].any()
    for k, v in auto.items():
        ref = r["ref64"][k][vis].reshape(v.shape)
        a = v.numpy()
        err = np.abs(ref - a)
        lim = 1e-10 * np.abs(a) + 1e-13 * np.abs(a).max()
        print(f"{k}: worst err / |autograd| {float((err / np.maximum(np.abs(a), 1e-300)).max()):.2e}")
        assert (err <= lim).all(), (k, float((err - lim).max()))


# ----------------------------------------------------------------------------------- correct implementations inside the budget
@pytest.mark.parametrize("name", list(pbc.SCENES))
def test_fp32_implementations_within_budget(shim, cases, name):
    """The C oracle (gcc -ffp-contract=off), the product's gms_preprocess.cuh built for the CPU, and a plain fp32 evaluation
    of the reference's tree each lie within the budget at every element of every visible Gaussian."""
    st, dg, r = cases[name]
    vis = st.radii > 0
    for k, v in r["budget"].items():
        assert np.isfinite(v).all() and np.isfinite(r["ref64"][k]).all(), k
    for impl, got in (("oracle", _oracle(st, dg)), ("hostshim", _shim(shim, st, dg)), ("fp32", _f32(st, dg))):
        for k, a in got.items():
            assert np.isfinite(a[vis]).all(), (impl, k)
        worst = _within(got, r, vis)
        print(f"[{name} {impl}] " + ", ".join(f"{k} {w:.3g}" for k, w in worst.items()))
        assert all(w <= 1.0 for w in worst.values()), (impl, worst)


def test_zero_record_has_zero_budget(shim, cases):
    """A zero record: budget 0 everywhere, and the implementations write exact zeros."""
    st, dg, _ = cases["deg3"]
    z = np.zeros_like(dg)
    r = preprocess64.preprocess_backward64(st, z)
    for k, v in r["budget"].items():
        assert not v.any() and not r["ref64"][k].any(), k
    for got in (_oracle(st, z), _shim(shim, st, z), _f32(st, z)):
        for k, a in got.items():
            assert not np.asarray(a).any(), k


# ----------------------------------------------------------------------------------------------------- the budget has teeth
SMALL = 1e-5


def _small(r, vis):
    """Visible Gaussians whose every gradient is below SMALL of the largest of its tensor: where a bug that reaches only
    some Gaussians (one branch, one lane, a term that matters only off the optical axis) hides from the global floor."""
    m = np.zeros(vis.shape[0])
    for k, v in r["ref64"].items():
        a = np.abs(v).reshape(v.shape[0], -1)
        if a.size and a.max() > 0:
            m = np.maximum(m, a.max(1) / a.max())
    return vis & (m > 0) & (m <= SMALL)


def _planted(st, dg, r, bug):
    """The fp32 evaluation with the bug on the small-gradient Gaussians, and whether the bug changes the operation there
    (its float64 evaluation differs from the reference at one of them)."""
    vis = st.radii > 0
    sel = _small(r, vis)
    vsel = sel[vis]
    _, I = preprocess64._inputs(st, dg)
    a, _ = preprocess64._evaluate(preprocess64._E64, I)
    b, _ = preprocess64._evaluate(preprocess64._E64, I, bug=bug)
    active = any(np.any((x.v != y.v) & vsel) for k in a for x, y in zip(a[k], b[k]))
    good, bad = _f32(st, dg), _f32(st, dg, bug)
    mixed = {}
    for k in good:
        m = sel.reshape((-1,) + (1,) * (np.ndim(good[k]) - 1))
        mixed[k] = np.where(m, bad[k], good[k])
    return mixed, active


@pytest.mark.parametrize("bug", preprocess64.BUGS)
def test_planted_bug_passes_old_floor_fails_budget(cases, bug):
    """Each bug, evaluated in fp32 on the Gaussians whose gradients are below 1e-5 of the largest: the old stage-2 floor
    passes it on at least one scene, and the per-element check rejects it on every scene where it changes the operation."""
    passed_floor, active = [], []
    for name, (st, dg, r) in cases.items():
        got, act = _planted(st, dg, r, bug)
        if not act:
            continue
        active.append(name)
        if _floor(got, _oracle(st, dg)):
            passed_floor.append(name)
        worst = _within(got, r, st.radii > 0)
        assert max(worst.values()) > 1.0, (name, worst)
    print(f"[{bug}] active on {len(active)} scenes: {active}; passes the old floor on {len(passed_floor)}: {passed_floor}")
    assert active and passed_floor, (bug, active, passed_floor)


# MEASURED (CPU, the scenes above, fp32 records of the C oracle's composite backward): the median of budget / |ref64| over
# nonzero elements is 1.7e-4 for the rotation gradient, 8.7e-5 for the scale gradient, 3.9e-5 for the covariance, 1.3e-5 for
# the mean, 1.1e-6 for SH and 0 for the pass-through outputs.  The bound leaves a factor of ~6 above the largest.
MEDIAN_MAX = 1e-3


def test_budget_not_vacuous(cases):
    tight = {}
    for name, (st, dg, r) in cases.items():
        for k, v in r["budget"].items():
            ref = np.abs(r["ref64"][k])
            nz = ref > 0
            if nz.any():
                tight.setdefault(k, []).append((v[nz] / ref[nz]))
    for k, parts in tight.items():
        a = np.concatenate(parts)
        med, p99 = float(np.median(a)), float(np.percentile(a, 99))
        print(f"[budget / |ref64|] {k}: median {med:.2e}, 99th percentile {p99:.2e} over {a.size} elements")
        assert med <= MEDIAN_MAX, (k, med)
