"""The composite forward per pixel: colour, inverse depth and final T of every pixel against a float64 evaluation of the same
operation, within an a-priori error budget; n_contrib among the values the flip candidates admit; the survivor lists equal to
the oracle's quad-hit mask (oracle.raster.composite_forward64; the derivation is next to gmso_composite_forward64 in
oracle/gms_oracle.c).

The global floor (1e-5 absolute on colour, inverse depth and final T, exact n_contrib) cannot see a dropped splat at a pixel
whose transmittance is already low: the pixel moves by T alpha |c - behind| and final T by T_final alpha / (1 - alpha), both
below 1e-5, and n_contrib does not move unless the splat was the last.  A 1e-5 error on a final T of 1e-4 is a 10 % error.

CPU: the fp32 oracle lies within the budget on every scene; the budget is far below the old floor where that floor is blind;
five plausible kernel bugs, built as mutated oracle runs, pass the old floor but fail the per-pixel check, and so does a NaN.
GPU (-m gpu): both forward kernels (2: scalar, 3: float2 pairs), forward-only and followed by a backward (fwd 2 then writes
survivor lists, which are compared)."""
import dataclasses

import numpy as np
import pytest

import raster_edge_cases as E
from gms_b200 import _lib
from gpu_helpers import assert_composite_forward_per_pixel, assert_forward_parity, run_gpu
from helpers import random_gaussians
from oracle import raster
from test_gpu_composite_budget import PARITY_SCENES, SCENES, _camera, _forward, _grads_in

OLD_TOL = 1e-5


def _edge(name):
    def build():
        S, g = E.CASES[name]()
        return S, g, E.oracle_forward(S, g)
    return build


def white_background():
    """A parity-suite scene on a white background: the T_final * bg term is as large as it gets."""
    S = _camera(320, 208, bg=(1.0, 1.0, 1.0))
    g = random_gaussians(3000, seed=3001, extent=1.2, scale_mu=-2.6)
    return S, g, _forward(S, g)


EDGE_SCENES = {f"edge_{k}": _edge(k) for k in E.CASES}
ALL_SCENES = {**SCENES, **PARITY_SCENES, **EDGE_SCENES}


def _outputs(st):
    return st.color, st.invdepth, st.final_T, st.n_contrib


def _old_floor_passes(st, color, invd, final_T, n_contrib):
    """The global check the parity helpers applied before: 1e-5 absolute on every output, n_contrib exact."""
    return bool(np.abs(color - st.color).max() <= OLD_TOL and np.abs(invd - st.invdepth).max() <= OLD_TOL
                and np.abs(final_T - st.final_T).max() <= OLD_TOL and (n_contrib == st.n_contrib).all())


def _new_check_passes(st, color, invd, final_T, n_contrib, r):
    try:
        assert_composite_forward_per_pixel(st, color, invd, final_T, n_contrib, r=r, label="mutated")
    except AssertionError as e:
        print(f"    rejected: {str(e)[:200]}")
        return False
    return True


# ------------------------------------------------------------------------------------------------------------ CPU: oracle
@pytest.mark.parametrize("name", list(ALL_SCENES))
def test_fp32_oracle_within_budget(name):
    """The fp32 oracle is an fp32 implementation of the operation: every pixel within the budget of the float64 reference,
    its own n_contrib admissible.  It performs the kernels' roundings in the same order (only its expf is more accurate than
    ex2.approx), so it sits closer to the bound than the backward oracle does to its own: measured <= 0.34 (final T on the
    deep translucent scene, whose thousand-splat chains round 1 - alpha the same way at every splat); 0.5 leaves the kernels'
    exp() error the other half."""
    S, g, st = ALL_SCENES[name]()
    r = raster.composite_forward64(st)
    worst = assert_composite_forward_per_pixel(st, *_outputs(st), r=r, label=f"oracle {name}")
    assert max(worst.values()) <= 0.5
    assert (r["adm"][..., 0] == st.n_contrib).all()
    cand, amb = r["cand"].astype(bool), st.ambiguous.astype(bool)
    print(f"[{name}] flip-candidate pixels {int(cand.sum())}, old fixed-band ambiguous pixels {int(amb.sum())}, "
          f"in both {int((cand & amb).sum())}")


def test_quad_hit_mask_matches_the_blend_decisions():
    """qhit: bit q of a list position set exactly when its splat blends at some pixel of quad q (an independent numpy
    evaluation of the fp32 decisions, away from the flip candidates)."""
    from test_gpu_composite_budget import _survivors_per_quad
    S, g, st = PARITY_SCENES["parity_3000"]()
    r = raster.composite_forward64(st)
    per_quad = []
    for (r0, r1) in st.ranges:
        h = r["qhit"][r0:r1]
        per_quad.extend(int(((h >> q) & 1).sum()) for q in range(4))
    ref = _survivors_per_quad(st)
    clean = np.array([not (r["qcand"][r0:r1] >> q & 1).any() for r0, r1 in st.ranges for q in range(4)])
    np.testing.assert_array_equal(np.array(per_quad)[clean], ref[clean])


@pytest.mark.parametrize("name", ["parity_3000", "saturating_30000", "partial_rounds", "deep_translucent"])
def test_budget_is_tight(name):
    """Median budget / |ref| per output, printed; on the low-T pixels (final T < 1e-3), where the old floor is blind, the
    median final T budget is at least 100x below 1e-5 and, on lists of hundreds, the median colour and inverse-depth
    budgets at least 2x below (they carry the rounding of every splat in front, about 100 u of the pixel's value).  The deep
    translucent scene's thousand-splat chains carry ten times that in colour: there only final T is held."""
    S, g, st = ALL_SCENES[name]()
    r = raster.composite_forward64(st)
    ref, bud = r["ref"], r["budget"]
    med = [float(np.median(bud[c][ref[c] != 0] / np.abs(ref[c][ref[c] != 0]))) for c in range(5)]
    low = st.final_T < 1e-3
    print(f"[{name}] median budget / |ref|: " + ", ".join(f"{k} {m:.2e}" for k, m in zip(raster.FWD64_OUTPUTS, med))
          + f"; low-T pixels {int(low.sum())} of {low.size}")
    assert low.sum() >= 100
    mlow = [float(np.median(bud[c][low])) for c in range(5)]
    print(f"[{name}] median budget on the low-T pixels: " + ", ".join(f"{k} {m:.2e}" for k, m in zip(raster.FWD64_OUTPUTS, mlow)))
    assert mlow[4] <= OLD_TOL / 100
    if name != "deep_translucent":
        assert max(mlow[:4]) <= OLD_TOL / 2
    assert all(m < 1e-3 for m in med)


# -------------------------------------------------------------------------------------------------- CPU: sensitivity
_SENS = {}


def _sens_case():
    """The 3000-splat parity scene (nearly opaque, many pixels with final T below 1e-3) and its reference and budget."""
    if not _SENS:
        S, g, st = PARITY_SCENES["parity_3000"]()
        _SENS.update(S=S, st=st, r=raster.composite_forward64(st))
    return _SENS


def _pixel_pairs(st, y, x):
    """The pairs that blend at pixel (x, y), front to back: (list position, Gaussian, alpha, T in front), numpy's fp32."""
    f32 = np.float32
    gx = (st.final_T.shape[1] + 15) // 16
    r0, _ = st.ranges[(y // 16) * gx + x // 16]
    T, out = 1.0, []
    for j in range(int(st.n_contrib[y, x])):
        i = int(st.point_list[r0 + j])
        dx, dy = f32(st.means2D[i, 0] - f32(x)), f32(st.means2D[i, 1] - f32(y))
        cx, cy, cz, op = st.conic_opacity[i]
        power = f32(-0.5) * (cx * dx * dx + cz * dy * dy) - cy * dx * dy
        if power > 0:
            continue
        a = float(min(0.99, op * np.exp(float(power))))
        if a < 1 / 255:
            continue
        out.append((j + 1, i, a, T))
        T *= 1 - a
    return out


def _clean_low_T_pixels(case, limit=1e-3):
    st, r = case["st"], case["r"]
    ys, xs = np.nonzero((st.final_T < limit) & ~r["cand"].astype(bool) & (st.ambiguous == 0) & (st.n_contrib > 3))
    return list(zip(ys.tolist(), xs.tolist()))


def _spliced(st, mutated, pixels):
    """The oracle's outputs with the mutated run's at `pixels` (a bug that reaches those pixels only)."""
    color, invd, fT, nc = (a.copy() for a in _outputs(st))
    for y, x in pixels:
        color[:, y, x] = mutated.color[:, y, x]; invd[:, y, x] = mutated.invdepth[:, y, x]
        fT[y, x] = mutated.final_T[y, x]; nc[y, x] = mutated.n_contrib[y, x]
    return color, invd, fT, nc


def _recomposite(st, **changes):
    m = dataclasses.replace(st, **changes)
    return raster.composite(m)


def test_sensitivity_reference_is_clean():
    """The unmutated fp32 oracle passes both checks (so a failure below is the mutation's)."""
    case = _sens_case()
    st = case["st"]
    assert _old_floor_passes(st, *_outputs(st)) and _new_check_passes(st, *_outputs(st), case["r"])


def test_sensitivity_dropped_pair():
    """One blended pair that is not the pixel's last dropped at a low-T pixel (a false negative of the quad cull)."""
    case = _sens_case()
    st = case["st"]
    for y, x in _clean_low_T_pixels(case)[::7][:60]:
        pairs = _pixel_pairs(st, y, x)
        if len(pairs) < 3:
            continue
        pos, i, a, T = pairs[-2]
        co = st.conic_opacity.copy()
        co[i, 3] = 0.0
        m = _recomposite(st, conic_opacity=co)
        out = _spliced(st, m, [(y, x)])
        if _old_floor_passes(st, *out):
            print(f"[dropped pair] pixel (x={x}, y={y}) position {pos}: T {T:.2e} alpha {a:.3f}")
            assert not _new_check_passes(st, *out, case["r"])
            return
    pytest.fail("no dropped pair passes the old floor")


def test_sensitivity_final_T_one_splat_early():
    """final T stored before the last blended splat's factor at a pixel whose last alpha is small."""
    case = _sens_case()
    st = case["st"]
    for y, x in _clean_low_T_pixels(case):
        pos, i, a, T = _pixel_pairs(st, y, x)[-1]
        if a > 0.1:
            continue
        color, invd, fT, nc = (v.copy() for v in _outputs(st))
        fT[y, x] = np.float32(st.final_T[y, x] / np.float32(1 - a))
        if _old_floor_passes(st, color, invd, fT, nc):
            print(f"[final T early] pixel (x={x}, y={y}): last alpha {a:.3f}, final T {st.final_T[y, x]:.3e} -> {fT[y, x]:.3e}")
            assert not _new_check_passes(st, color, invd, fT, nc, case["r"])
            return
    pytest.fail("no pixel with a small last alpha")


def test_sensitivity_last_partial_round_skipped():
    """A quad's last partial 32-splat round skipped at the pixels whose T is below 1e-3 when it starts: its blends are lost
    while its splats are still counted in n_contrib (the count and the blend are separate updates in the kernels)."""
    case = _sens_case()
    st = case["st"]
    H, W = st.final_T.shape
    gx = (W + 15) // 16
    for t in np.argsort(-(st.ranges[:, 1] - st.ranges[:, 0])):
        r0, r1 = (int(v) for v in st.ranges[t])
        n = r1 - r0
        if n <= 32 or n % 32 == 0:
            continue
        base = (n - 1) // 32 * 32
        rng = st.ranges.copy()
        rng[t, 1] = r0 + base
        m = _recomposite(st, ranges=rng)
        y0, x0 = (t // gx) * 16, (t % gx) * 16
        for q in range(4):
            ys, xs = np.mgrid[y0 + (q >> 1) * 8: min(y0 + (q >> 1) * 8 + 8, H), x0 + (q & 1) * 8: min(x0 + (q & 1) * 8 + 8, W)]
            pix = [(y, x) for y, x in zip(ys.ravel(), xs.ravel()) if m.final_T[y, x] < 1e-3]
            if not pix:
                continue
            out = _spliced(st, m, pix)[:3] + (st.n_contrib,)
            if (out[0] != st.color).any() and _old_floor_passes(st, *out):
                print(f"[partial round] tile {t} quad {q}: list {n}, round from {base} skipped at {len(pix)} pixels")
                assert not _new_check_passes(st, *out, case["r"])
                return
    pytest.fail("no partial round whose loss passes the old floor")


def test_sensitivity_background_with_earlier_transmittance():
    """The background FMA using the transmittance in front of the last blended splat instead of behind it."""
    case = _sens_case()
    st = case["st"]
    bg = np.asarray(st.settings.bg, np.float32)
    best = None
    for y, x in _clean_low_T_pixels(case):
        a = _pixel_pairs(st, y, x)[-1][2]
        Tprev = np.float32(st.final_T[y, x] / np.float32(1 - a))
        d = float((Tprev - st.final_T[y, x]) * bg.max())
        if d <= 0.8 * OLD_TOL and (best is None or d > best[0]):
            best = (d, y, x, a, Tprev)
    assert best is not None, "no pixel whose background change stays below the old floor"
    d, y, x, a, Tprev = best          # the largest change the old floor cannot see
    color, invd, fT, nc = (v.copy() for v in _outputs(st))
    color[:, y, x] = color[:, y, x] + (Tprev - st.final_T[y, x]) * bg
    print(f"[background] pixel (x={x}, y={y}): last alpha {a:.3f}, T {st.final_T[y, x]:.3e} -> {Tprev:.3e}")
    assert _old_floor_passes(st, color, invd, fT, nc)
    assert not _new_check_passes(st, color, invd, fT, nc, case["r"])


def test_sensitivity_relative_error_in_G():
    """A 1e-4 relative error in G = exp(power) of one splat, at every pixel it reaches (alpha = op * G: the opacity scaled)."""
    case = _sens_case()
    st = case["st"]
    vis = np.flatnonzero((st.radii > 0) & (st.conic_opacity[:, 3] >= 0.5) & (st.conic_opacity[:, 3] < 0.9))
    rs = np.random.RandomState(5)
    for i in rs.permutation(vis)[:40]:
        co = st.conic_opacity.copy()
        co[i, 3] = np.float32(co[i, 3] * (1 + 1e-4))
        m = _recomposite(st, conic_opacity=co)
        out = _outputs(m)
        if (m.final_T != st.final_T).any() and _old_floor_passes(st, *out):
            print(f"[G error] Gaussian {i}: {int((m.final_T != st.final_T).sum())} pixels move")
            assert not _new_check_passes(st, *out, case["r"])
            return
    pytest.fail("no splat whose G error passes the old floor")


@pytest.mark.parametrize("out", ["color", "invdepth", "final_T"])
def test_nan_fails(out):
    """A NaN in any output fails, also at a pixel nothing blends into (the grazing mesh scene has such pixels: budget from
    the background term alone)."""
    S, g, st = SCENES["flat_mesh_grazing"]()
    r = raster.composite_forward64(st)
    empty, busy = np.argwhere(st.n_contrib == 0), np.argwhere(st.n_contrib > 0)
    assert empty.shape[0] and busy.shape[0]
    assert _new_check_passes(st, *_outputs(st), r)
    for y, x in (empty[0], busy[0]):
        color, invd, fT, nc = (v.copy() for v in _outputs(st))
        {"color": color[1], "invdepth": invd[0], "final_T": fT}[out][y, x] = np.nan
        assert not _new_check_passes(st, color, invd, fT, nc, r)


# ----------------------------------------------------------------------------------------------------------------- GPU
GPU_SCENES = {**SCENES, **PARITY_SCENES, "antialiasing": _edge("antialiasing"), "white_background": white_background}
MAX_AMBIGUOUS = {"deep_translucent": 0.02}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["forward_only", "with_backward"])
@pytest.mark.parametrize("fwd", [2, 3])
@pytest.mark.parametrize("name", list(GPU_SCENES))
def test_gpu_composite_forward_within_budget(name, fwd, mode):
    S, g, st = GPU_SCENES[name]()
    dC, dI = _grads_in(st) if mode == "with_backward" else (None, None)
    old = _lib.set_option("composite_fwd", fwd)
    try:
        color, radii, invd, state, _ = run_gpu(S, g, dC, dI)
    finally:
        _lib.set_option("composite_fwd", old)
    lists = fwd == 2 and mode == "with_backward"
    assert ("surv" in state) == lists, "survivor lists present exactly when fwd 2 runs ahead of a backward"
    print(f"[{name} fwd{fwd} {mode}]", end=" ")
    worst = assert_forward_parity(st, color, radii, invd, state, max_ambiguous=MAX_AMBIGUOUS.get(name, 5e-4))
    assert set(worst) == {"r", "g", "b", "invdepth", "final_T"}
