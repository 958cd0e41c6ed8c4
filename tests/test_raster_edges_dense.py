"""The C oracle against the independent float64 autograd model (oracle/torch_dense.py) on the edge scenes of
tests/raster_edge_cases.py: near plane, guard band, off-screen and int32-sized footprints, screen-filling splats, the
antialiasing floor, SH clamping along every axis, opacity limits, exact pixel / quad / tile positions, depth ties and ragged
images.  Forward and every gradient.

Upstream gradients are zeroed at the oracle's threshold-ambiguous pixels, so both models blend the same splats wherever the
gradient is compared.  The sliver sweep is not here: its fp32 quadratic form cancels, so float64 is the wrong yardstick
(it is checked GPU against oracle, tests/test_gpu_raster_edges.py)."""
import numpy as np
import pytest
import torch

import raster_edge_cases as E
from oracle import raster, torch_dense

# per case: (forward abs tolerance per pixel, gradient max err / max |ref|).  Every case measured <= 4.3e-6 forward and
# <= 6.9e-6 for any gradient (ragged 93x61: rotations), so one bound of 2e-5 / 1e-4 holds them all with a 3x / 14x margin.
TOL = {}
DEFAULT_TOL = (2e-5, 1e-4)


def dense_case(S, g, seed=0):
    """Oracle forward + backward and the dense model's forward + autograd backward on the same upstream gradients (zero at the
    oracle's ambiguous pixels).  Returns (st, oracle grads, dense tensors, dense outputs)."""
    st = E.oracle_forward(S, g)
    H, W = S.image_height, S.image_width
    rs = np.random.RandomState(seed + 100)
    ok = st.ambiguous == 0
    dC = (rs.randn(3, H, W) * ok).astype(np.float32)
    dI = (rs.randn(H, W) * ok).astype(np.float32)
    grads = raster.backward(st, dC, dI)
    # the dense model gets the drawn splats only: a culled one at depth 0 would put inf * 0 into its autograd graph
    vis = st.radii > 0
    kw = {k: v[torch.from_numpy(vis)] for k, v in g.items() if v is not None}
    t = {k: v.double().clone().requires_grad_(True) for k, v in kw.items()}
    sink = torch.zeros(int(vis.sum()), 3, dtype=torch.float64, requires_grad=True)
    color, invd, final_T, n_contrib = torch_dense.render(
        S, st.rects[vis], t["means3D"], sink, t["opacities"], shs=t.get("shs"), colors_precomp=t.get("colors_precomp"),
        scales=t.get("scales"), rotations=t.get("rotations"), cov3D_precomp=t.get("cov3D_precomp"), depths32=st.depths[vis])
    loss = (color * torch.tensor(dC, dtype=torch.float64)).sum() + (invd[0] * torch.tensor(dI, dtype=torch.float64)).sum()
    loss.backward()
    return st, grads, t, sink, (color.detach().numpy(), invd.detach().numpy(), final_T.detach().numpy(), n_contrib.numpy()), (dC, dI)


GRAD_PAIRS = [("means3D", "dL_dmeans3D"), ("opacities", "dL_dopacity"), ("shs", "dL_dsh"), ("scales", "dL_dscales"),
              ("rotations", "dL_drotations")]


def _rel(a, b):
    a = np.asarray(a, np.float64).reshape(-1)
    b = np.asarray(b, np.float64).reshape(-1)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def check_against_dense(name, S, g, seed=0):
    ftol, gtol = TOL.get(name, DEFAULT_TOL)
    st, grads, t, sink, (color, invd, final_T, n_contrib), _ = dense_case(S, g, seed)
    ok = st.ambiguous == 0
    np.testing.assert_array_equal(st.n_contrib[ok], n_contrib[ok])
    fe = max(float(np.abs(st.color - color)[:, ok].max()), float(np.abs(st.invdepth - invd)[:, ok].max()),
             float(np.abs(st.final_T - final_T)[ok].max()))
    vis = st.radii > 0
    errs = {"means2D": _rel(grads["dL_dmeans2D"][vis, :2], sink.grad[:, :2])}
    for kt, kr in GRAD_PAIRS:
        if kt in t and grads.get(kr) is not None:
            errs[kt] = _rel(grads[kr][vis], t[kt].grad)
            assert not np.any(grads[kr][~vis]), f"{name}: culled splats must get zero {kr}"
    print(f"[dense {name}] {S.image_width}x{S.image_height} P={st.radii.shape[0]} N={st.N} ambiguous={int((~ok).sum())} "
          f"forward max|oracle-dense| {fe:.1e} (tol {ftol:.0e}); grads max err/max|ref| (tol {gtol:.0e}): " +
          ", ".join(f"{k} {e:.1e}" for k, e in errs.items()))
    assert fe <= ftol, (name, fe)
    for k, e in errs.items():
        assert e <= gtol, (name, k, e)
    return st, grads, errs


@pytest.mark.parametrize("name", list(E.CASES))
def test_oracle_matches_dense_model_on_edge_case(name):
    S, g = E.CASES[name]()
    check_against_dense(name, S, g)


def test_near_plane_cull_and_mark_visible():
    """`<=`: exactly 0.2 is culled, the next float above it is drawn; markVisible says the same."""
    S, g = E.near_plane()
    st = E.oracle_forward(S, g)
    z = g["means3D"][:, 2].numpy()
    vis = raster.mark_visible(S, g["means3D"])
    assert not vis[0] and vis[2] and st.radii[0] == 0 and st.radii[2] > 0
    np.testing.assert_array_equal(vis, st.radii > 0)
    np.testing.assert_array_equal(vis, z > E.NEAR)


def test_saturating_float_to_int_conversion():
    """The oracle's float -> int32 conversion has the device's cvt.rzi.s32.f32 semantics."""
    f = raster.f2i_sat
    assert f(float("nan")) == 0 and f(float("inf")) == 2 ** 31 - 1 and f(float("-inf")) == -2 ** 31
    assert f(3e9) == 2 ** 31 - 1 and f(-3e9) == -2 ** 31 and f(2147483520.0) == 2147483520
    assert f(2147483648.0) == 2 ** 31 - 1 and f(-2147483648.0) == -2 ** 31
    assert f(-2.7) == -2 and f(2.7) == 2 and f(-0.5) == 0


def test_radius_beyond_int32_covers_the_whole_grid():
    """A footprint of ~8e9 px: radius saturates to INT32_MAX, the rect is the whole grid, and the splat is composited into
    every tile; a centre ~1e11 px off-screen saturates its rect bounds and is culled."""
    S, g = E.offscreen()
    st = E.oracle_forward(S, g)
    n = st.radii.shape[0] - 2
    T = st.ranges.shape[0]
    assert st.radii[n] == E.INT32_MAX and st.tiles_touched[n] == T
    assert all(n in st.point_list[st.ranges[t, 0]:st.ranges[t, 1]] for t in range(T))
    assert st.radii[n + 1] == 0 and st.tiles_touched[n + 1] == 0


def test_sliver_sweep_reaches_large_terms():
    """The sweep's regime: blending pixels whose quadratic-form terms reach >= 1e6 (asserted by the builder); reported here."""
    cases = E.sliver_sweep()
    assert len(cases) == len(E.SLIVER_SIGMAS) * len(E.SLIVER_MINORS) * 2 * 24
    print("[sliver sweep] largest term magnitude S at a blending pixel, per major sigma: " +
          ", ".join(f"{s} px: {v:.2e}" for s, v in sorted(E.sliver_sweep.smax.items())))
