"""-m gpu: the CUDA rasterizer against the C oracle (and, on the small scenes, the float64 dense model) on the edge scenes
of tests/raster_edge_cases.py, under every composite option; the composite kernels' quad cull on the sliver sweep; and one
sync-free free-Gaussian training frame with the camera inside the point cloud."""
import numpy as np
import pytest
import torch

import raster_edge_cases as E
from gms_b200 import scenes
from gpu_helpers import run_gpu, assert_forward_parity, assert_grad_parity
from oracle import raster
from test_gpu_free_train import BG, LAMBDA, RAW_TOL, _Options, _grads, _gt, _model, _oracle_raw, _views
from test_raster_edges_dense import dense_case

pytestmark = pytest.mark.gpu

COMPOSITE = [(2, 5), (2, 3), (3, 3), (3, 5)]       # (composite_fwd, composite_bwd); fwd 3 writes no survivor lists: bwd 3 runs


def _upstream(st, seed=1):
    """Random upstream gradients, zero at the oracle's threshold-ambiguous pixels (where exp() may flip a skip decision)."""
    H, W = st.final_T.shape
    rs = np.random.RandomState(seed)
    ok = st.ambiguous == 0
    return (rs.randn(3, H, W) * ok).astype(np.float32), (rs.randn(H, W) * ok).astype(np.float32)


@pytest.mark.parametrize("fwd,bwd", COMPOSITE)
@pytest.mark.parametrize("name", list(E.CASES))
def test_gpu_matches_oracle_on_edge_case(name, fwd, bwd):
    """Integers bit-exact, image <= 1e-5 outside the ambiguous pixels, gradients at the staged tolerances."""
    S, g = E.CASES[name]()
    st = E.oracle_forward(S, g)
    dC, dI = _upstream(st)
    gref = raster.backward(st, dC, dI)
    with _Options({"composite_fwd": fwd, "composite_bwd": bwd}):
        color, radii, invd, state, grads = run_gpu(S, g, dC, dI)
    print(f"[edge {name} fwd{fwd} bwd{bwd}]", end=" ")
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(grads, gref, st=st)


def test_gpu_radius_beyond_int32_saturates_like_the_oracle():
    """The device's float -> int conversion saturates: radius INT32_MAX, a whole-grid rect; a centre whose rect bounds exceed
    int32 is culled.  The oracle's conversion gives the same."""
    S, g = E.offscreen()
    st = E.oracle_forward(S, g)
    color, radii, invd, state, _ = run_gpu(S, g)
    n = radii.shape[0] - 2
    T = st.ranges.shape[0]
    assert radii[n] == E.INT32_MAX == st.radii[n] and int(state["tiles_touched"][n]) == T
    assert radii[n + 1] == 0 == st.radii[n + 1]
    assert_forward_parity(st, color, radii, invd, state)


def test_gpu_mark_visible_at_the_near_plane():
    import diff_gaussian_rasterization as dgr
    from gpu_helpers import gpu_settings
    S, g = E.near_plane()
    vis = dgr.GaussianRasterizer(raster_settings=gpu_settings(S)).markVisible(g["means3D"].cuda()).cpu().numpy()
    np.testing.assert_array_equal(vis, raster.mark_visible(S, g["means3D"]))
    np.testing.assert_array_equal(vis, g["means3D"][:, 2].numpy() > E.NEAR)


# GPU against the float64 dense model directly: every gradient measured <= 5.1e-6 of max on an H100 (ragged 93x61, rotations);
# the bound is the oracle-vs-dense one
DENSE_GPU_TOL = 1e-4


@pytest.mark.parametrize("name", list(E.CASES))
def test_gpu_matches_dense_model_on_edge_case(name):
    S, g = E.CASES[name]()
    st, _, t, sink, (color_d, invd_d, final_T_d, n_contrib_d), (dC, dI) = dense_case(S, g)
    color, radii, invd, state, grads = run_gpu(S, g, dC, dI)
    ok = st.ambiguous == 0
    np.testing.assert_array_equal(state["n_contrib"][ok], n_contrib_d[ok])
    fe = max(float(np.abs(color - color_d)[:, ok].max()), float(np.abs(invd - invd_d)[:, ok].max()),
             float(np.abs(state["final_T"] - final_T_d)[ok].max()))
    vis = radii > 0
    errs = {"means2D": float(np.abs(grads["means2D"][vis, :2] - sink.grad.numpy()[:, :2]).max() / np.abs(sink.grad.numpy()[:, :2]).max())}
    for k in ("means3D", "opacities", "shs", "scales", "rotations"):
        ref = t[k].grad.numpy().reshape(-1)
        errs[k] = float(np.abs(grads[k][vis].reshape(-1) - ref).max() / max(np.abs(ref).max(), 1e-30))
        assert not np.any(grads[k][~vis])
    print(f"[gpu vs dense {name}] forward {fe:.1e}; grads " + ", ".join(f"{k} {e:.1e}" for k, e in errs.items()))
    assert fe <= 2e-5
    for k, e in errs.items():
        assert e <= DENSE_GPU_TOL, (k, e)


@pytest.mark.parametrize("fwd", [2, 3])
def test_quad_cull_keeps_every_blending_pixel_of_slivers(fwd):
    """The sliver sweep, one splat per frame: n_contrib bit-exact and the image within 1e-5 outside the ambiguous pixels.  A
    quad the cull skips although one of its pixels blends under the canonical per-pixel sequence shows up as a pixel with
    n_contrib 0 on the GPU and 1 in the oracle.  Mismatches are counted per major sigma before anything is asserted."""
    bad, amb, worst = {}, {}, 0.0
    with _Options({"composite_fwd": fwd}):
        for tag, S, g in E.sliver_sweep():
            sigma = int(tag.split("-")[0][5:])
            st = E.oracle_forward(S, g)
            color, radii, invd, state, _ = run_gpu(S, g)
            np.testing.assert_array_equal(radii, st.radii)
            ok = st.ambiguous == 0
            wrong = int((state["n_contrib"][ok] != st.n_contrib[ok]).sum())
            bad[sigma] = bad.get(sigma, 0) + wrong
            amb[sigma] = amb.get(sigma, 0) + int((~ok).sum())
            if not wrong:
                worst = max(worst, float(np.abs(color - st.color)[:, ok].max()))
    print(f"[sliver cull fwd{fwd}] pixels with a wrong n_contrib per major sigma: {bad}; ambiguous pixels: {amb}; "
          f"max|image-oracle| where n_contrib agrees: {worst:.1e}; largest S at a blending pixel: "
          + ", ".join(f"{s}: {v:.2e}" for s, v in sorted(E.sliver_sweep.smax.items())))
    assert sum(bad.values()) == 0, bad
    assert worst <= 1e-5


def _sliver_term_magnitudes(st, dC, dI):
    """Sum over the blending pixels of the magnitude of each per-pixel term of the composite backward's per-Gaussian sums, for
    a one-splat frame (float64).  For a sliver the terms of dL/dmean2D are G (cx dx + cy dy) with |cx dx| ~ 1e4 that cancel
    from pixel to pixel, so an fp32 sum (GPU) and a double sum of fp32 terms (oracle) differ by ~2^-24 of this magnitude,
    not of the result."""
    i = int(np.flatnonzero(st.radii > 0)[0])
    ys, xs = np.nonzero(st.n_contrib > 0)
    cx, cy, cz, op = (float(v) for v in st.conic_opacity[i])
    f32 = np.float32
    dx32 = (st.means2D[i, 0] - xs.astype(f32)).astype(f32)
    dy32 = (st.means2D[i, 1] - ys.astype(f32)).astype(f32)
    fma = lambda a, b, c: (a.astype(np.float64) * b + c).astype(f32)        # fp32 a*b is exact in float64
    c32 = st.conic_opacity[i].astype(f32)
    # G from the canonical fp32 power the kernels and the oracle blend with: for these slivers it differs from the exact
    # form by thousands, so a float64 G would weigh the wrong pixels
    t = fma(c32[2] * dy32, dy32, (c32[0] * dx32) * dx32)
    power = fma(-(c32[1] * dx32), dy32, f32(-0.5) * t)
    G = np.exp(power.astype(np.float64))
    dx, dy = dx32.astype(np.float64), dy32.astype(np.float64)
    alpha = np.minimum(0.99, op * G)
    bg = np.asarray(st.settings.bg, np.float64)
    dpix = dC[:, ys, xs].astype(np.float64)
    da = (np.abs(st.rgb[i][:, None] * dpix).sum(0) + np.abs(dI[ys, xs] / st.depths[i])
          + np.abs((bg[:, None] * dpix).sum(0)) / (1 - alpha))
    dG = op * da
    W, H = st.settings.image_width, st.settings.image_height
    return {"dL_dmean2D": np.array([(dG * G * (abs(cx * dx) + abs(cy * dy))).sum() * 0.5 * W,
                                    (dG * G * (abs(cz * dy) + abs(cy * dx))).sum() * 0.5 * H]),
            "dL_dconic": 0.5 * np.array([(G * dG * dx * dx).sum(), (G * dG * abs(dx * dy)).sum(), (G * dG * dy * dy).sum()]),
            "dL_dopacity": np.array([(G * da).sum()]),
            "dL_dcolor": (alpha[None] * np.abs(dpix)).sum(1)}


@pytest.mark.parametrize("fwd,bwd", [(2, 5), (2, 3)])
def test_sliver_backward_matches_oracle(fwd, bwd):
    """The backward over the same slivers: the composite backward's per-Gaussian sums against the oracle's double-accumulated
    ones (bwd 3 re-derives the survivors with the same cull), each within 16 * 2^-24 of the magnitude it is summed from
    (_sliver_term_magnitudes; measured <= 2.0 on an H100).  A pixel the backward skipped would move a sum by one whole term, ~1e-3 of that magnitude
    for the few hundred pixels a sliver blends.  A subset: sigma 1500 and 6000, off-screen centres."""
    worst = {}
    with _Options({"composite_fwd": fwd, "composite_bwd": bwd}):
        for tag, S, g in E.sliver_sweep():
            if not (tag.startswith(("sigma1500-", "sigma6000-")) and "-off-" in tag):
                continue
            st = E.oracle_forward(S, g)
            if not (st.n_contrib > 0).any():
                continue
            dC, dI = _upstream(st)
            gref = raster.backward(st, dC, dI)
            color, radii, invd, state, grads = run_gpu(S, g, dC, dI)
            dg, comp = grads["_dgeom"], gref["_composite"]
            i = int(np.flatnonzero(st.radii > 0)[0])
            mag = _sliver_term_magnitudes(st, dC, dI)
            for k, sl in (("dL_dmean2D", slice(0, 2)), ("dL_dconic", slice(2, 5)), ("dL_dopacity", slice(5, 6)),
                          ("dL_dcolor", slice(6, 9))):
                ref = np.asarray(comp[k], np.float64).reshape(dg.shape[0], -1)[i]
                e = float((np.abs(dg[i, sl] - ref) / (2.0 ** -24 * mag[k] + 1e-30)).max())
                worst[k] = max(worst.get(k, 0.0), e)
    print(f"[sliver backward fwd{fwd} bwd{bwd}] composite backward max |gpu - oracle| in units of 2^-24 x term magnitude: " +
          ", ".join(f"{k} {e:.1f}" for k, e in worst.items()))
    for k, e in worst.items():
        assert e <= 16, (k, e)


# ------------------------------------------------------------------------------ one sync-free frame, camera inside the cloud
def _inside_raw(P=3000, seed=13):
    from helpers import random_gaussians
    g = random_gaussians(P, seed=seed, extent=2.0, scale_mu=-3.2, flat_frac=0.0)
    gen = torch.Generator().manual_seed(seed + 1)
    rot = g["rotations"] * (0.5 + torch.rand(P, 1, generator=gen))
    s = torch.log(g["scales"])[:, 1:].contiguous()
    return dict(xyz=g["means3D"], scaling=s, rotation=rot, features=g["shs"], opacity=torch.logit(g["opacities"]))


@pytest.mark.parametrize("opts", [{}, {"bin_impl": 1}], ids=["defaults", "bin_impl=1"])
def test_free_frame_with_the_camera_inside_the_cloud(opts):
    """gms_free_train_frame (NativeFreeFrame, gs_flat) on a camera near the centre of a 3k-point cloud of extent 2: splats
    behind the camera, at the near plane, beyond the guard band and hundreds of pixels wide are all in the frame.  Its second
    (sync-free) run against the oracle chain, as tests/test_gpu_free_train.py checks the ordinary scenes."""
    import aten_reference
    from gpu_helpers import assert_image_parity
    from helpers import settings_from_camera
    W, H = 320, 240
    raw = _inside_raw()
    cam0 = scenes.look_at_camera((0.05, -0.03, 0.02), (1.0, 0.3, -0.2), W, H)
    S = settings_from_camera(cam0, sh_degree=3, bg=BG)
    # regime: the frame holds splats behind / at the near plane / past the guard band / with wide footprints
    m3 = raw["xyz"].numpy().astype(np.float32)
    view = np.asarray(S.viewmatrix, np.float32).reshape(4, 4)
    pv = m3 @ view[:3, :3] + view[3, :3]
    z = pv[:, 2]
    assert (z <= 0).sum() > 500 and ((z > 0.2) & (z < 0.3)).sum() >= 3
    assert (np.abs(pv[:, 0] / np.where(z > 0.2, z, np.inf)) > 1.3 * S.tanfovx).sum() > 100
    cam, gt, bg = cam0.to("cuda"), _gt(3, W, H).cuda(), torch.tensor(BG, device="cuda")
    with _Options(opts):
        from gms_b200.trainer import NativeFreeFrame
        m, _ = _model(raw, "gs_flat", 3)
        fr = NativeFreeFrame(m, W, H, LAMBDA)
        fr.run(cam, gt, bg, stats=False)
        loss = float(fr.run(cam, gt, bg, stats=False))
        torch.cuda.synchronize()
        assert fr.overflows == 0
        out = _views(fr, m.P)
    img = out["image"].cpu().double().requires_grad_(True)
    aten_reference.training_loss(img, gt.cpu().double(), LAMBDA).backward()
    st, og = _oracle_raw(raw, "gs_flat", out, img.grad.float().numpy(), S)
    np.testing.assert_array_equal(out["radii"].cpu().numpy(), st.radii)
    assert fr.last_num_rendered == st.N
    assert int(st.radii.max()) > 200
    assert_image_parity(st, out["image"].cpu().numpy())
    ref_loss = float(aten_reference.training_loss(torch.tensor(st.color, dtype=torch.float64), gt.cpu().double(), LAMBDA))
    assert abs(loss - ref_loss) <= 1e-5 * max(1.0, abs(ref_loss))
    got = _grads(m)
    errs = {k: float((got[k].cpu().double().reshape(ref.shape) - ref).abs().max()) / max(float(ref.abs().max()), 1e-20)
            for k, ref in og.items()}
    print(f"[free frame inside the cloud {opts}] P={m.P} N={st.N} visible={int((st.radii > 0).sum())} max radius "
          f"{int(st.radii.max())} grad err/max: " + ", ".join(f"{k} {e:.2e}" for k, e in errs.items()))
    for k, e in errs.items():
        assert e <= RAW_TOL[k], (k, e)
