"""Deterministic rasterizer scenes at the edges the benign parity scenes never reach (CPU builders, oracle side).

Every builder returns `(Settings, inputs)` (or, for the sweeps, a list of `(tag, Settings, inputs)`) and asserts, with the C
oracle, that its scene is in the regime its name promises: a test that silently stopped reaching its edge would still pass.

Most scenes use `camera()`: identity rotation at the origin, so view space is world space and the depth of a Gaussian is
its z, bit for bit.  Positions that must land exactly on a pixel are found by `snap`, which replays the fp32
projection sequence of the oracle and the kernels over neighbouring floats of x, y and z until the pixel is hit exactly.
"""
from __future__ import annotations

import functools
import math

import numpy as np
import torch

from gms_b200 import scenes
from helpers import settings_from_camera, random_gaussians
from oracle import raster

NEAR = np.float32(0.2)
INT32_MAX = 2 ** 31 - 1
SLIVER_SIGMAS = (500, 1500, 3000, 6000)
SLIVER_MINORS = (2e-8, 0.0)
AA_FLOOR = 0.000025


def camera(W, H, R=None, eye=(0.0, 0.0, 0.0), fovx=scenes.NERF_FOVX):
    """A scenes.Camera at `eye` with world->view rotation R (rows: right, down, forward); identity by default."""
    R = np.eye(3) if R is None else np.asarray(R, np.float64)
    eye = np.asarray(eye, np.float64)
    Rt = np.eye(4)
    Rt[:3, :3] = R
    Rt[:3, 3] = -R @ eye
    wvt = torch.tensor(np.float32(Rt)).transpose(0, 1).contiguous()
    focal = W / (2 * math.tan(fovx / 2))
    fovy = 2 * math.atan(H / (2 * focal))
    proj = scenes.projection_matrix(scenes.ZNEAR, scenes.ZFAR, fovx, fovy).transpose(0, 1)
    full = (wvt.unsqueeze(0).bmm(proj.unsqueeze(0))).squeeze(0).contiguous()
    return scenes.Camera(W, H, fovx, fovy, wvt, full, wvt.inverse()[3, :3].contiguous())


def settings(W, H, sh_degree=3, antialiasing=False, bg=(0.1, 0.4, 0.8), **kw):
    return settings_from_camera(camera(W, H, **kw), sh_degree=sh_degree, bg=bg, antialiasing=antialiasing)


def focal(S):
    return float(np.float32(S.image_width) / (np.float32(2.0) * np.float32(S.tanfovx)))


def _pix(S, v, z, axis):
    """Pixel coordinate of view-space coordinate v (float32 array) at depth z under camera(): the oracle's fp32 sequence."""
    f32 = np.float32
    m = f32(np.asarray(S.projmatrix, np.float32).reshape(16)[0 if axis == 0 else 5])
    n = f32(S.image_width if axis == 0 else S.image_height)
    ph = (m * np.asarray(v, np.float32)).astype(np.float32)
    pw = f32(1.0) / (f32(z) + f32(1e-7))
    pp = (ph * pw).astype(np.float32)
    a = (pp + f32(1.0)).astype(np.float32)
    return (np.float32(a.astype(np.float64) * float(n) - 1.0) * f32(0.5)).astype(np.float32)


def _hits(S, target, zs, axis):
    """For each candidate depth, the fp32 view coordinate nearest the float64 inverse that projects exactly onto `target`
    (NaN where none within 256 ulps does).  The projection has ~32x coarser steps than the pixel coordinate's ulp, so
    only some depths admit an exact hit."""
    n = S.image_width if axis == 0 else S.image_height
    t = S.tanfovx if axis == 0 else S.tanfovy
    v0 = (((2.0 * target + 1.0) / n - 1.0) * t * (zs.astype(np.float64) + 1e-7)).astype(np.float32)
    step = np.spacing(np.maximum(np.abs(v0), np.float32(1e-6)))
    cand = (v0[:, None] + np.arange(-256, 257)[None, :] * step[:, None]).astype(np.float32)
    ok = _pix(S, cand, zs[:, None], axis) == np.float32(target)
    dist = np.where(ok, np.abs(cand.astype(np.float64) - v0[:, None]), np.inf)
    best = dist.argmin(1)
    return np.where(ok.any(1), cand[np.arange(len(zs)), best], np.nan)


def snap(S, px, py, z):
    """(x, y, z') under camera(), z' within a few thousand ulps of z, whose fp32 projection is exactly pixel (px, py)."""
    z0 = np.float32(z)
    zs = (z0 + np.arange(-4000, 4001) * np.spacing(z0)).astype(np.float32)
    zs = zs[np.argsort(np.abs(zs - z0), kind="stable")]
    hx, hy = _hits(S, px, zs, 0), _hits(S, py, zs, 1)
    ok = np.flatnonzero(~np.isnan(hx) & ~np.isnan(hy))
    assert ok.size, f"no fp32 position projects exactly onto pixel ({px}, {py}) near depth {z}"
    i = ok[0]
    return float(hx[i]), float(hy[i]), float(zs[i])


def unproject(S, px, py, z):
    """Approximate inverse of the projection of camera() (float64): view-space (x, y) of pixel (px, py) at depth z."""
    return ((2.0 * px + 1.0) / S.image_width - 1.0) * S.tanfovx * z, ((2.0 * py + 1.0) / S.image_height - 1.0) * S.tanfovy * z


def random_quats(P, rs):
    q = rs.randn(P, 4)
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def z_quat(theta):
    """Rotation about the view axis by theta: columns of R are (cos, sin, 0), (-sin, cos, 0), (0, 0, 1)."""
    return np.array([math.cos(theta / 2), 0.0, 0.0, math.sin(theta / 2)])


def shs_for(rgb, rs, rest=0.1):
    """SH rows [P,16,3] whose DC term gives colour `rgb` [P,3] (before the other bands) and small random higher bands."""
    rgb = np.asarray(rgb, np.float64)
    dc = (rgb - 0.5) / scenes.SH_C0
    return np.concatenate([dc[:, None, :], rest * rs.randn(rgb.shape[0], 15, 3)], 1)


def make_inputs(xyz, scales, quats, opac, shs):
    t = lambda a: torch.tensor(np.asarray(a, np.float32))
    return dict(means3D=t(xyz), scales=t(scales), rotations=t(quats), opacities=t(np.reshape(opac, (-1, 1))),
                shs=t(shs).contiguous())


def oracle_forward(S, g):
    return raster.forward(S, g["means3D"], g["opacities"], shs=g.get("shs"), colors_precomp=g.get("colors_precomp"),
                          scales=g.get("scales"), rotations=g.get("rotations"), cov3D_precomp=g.get("cov3D_precomp"))


# ------------------------------------------------------------------------------------------------------------ builders
def near_plane():
    """Depths exactly 0.2 (culled: the test is `<=`), the next float above, 0.2005, 0.21, 0.25, and 0 / -0.1 (behind)."""
    S = settings(96, 64)
    rs = np.random.RandomState(1)
    depths = [NEAR, np.nextafter(NEAR, np.float32(1)), np.float32(0.2005), np.float32(0.21), np.float32(0.25),
              np.float32(0.0), np.float32(-0.1)]
    xyz, sc = [], []
    for i, z in enumerate(depths):
        for j in range(2):
            px, py = 10 + 12 * i + rs.uniform(0, 3), 18 + 26 * j + rs.uniform(0, 3)
            zz = max(float(z), 0.2)
            x, y = unproject(S, px, py, zz)
            xyz.append((x, y, z))
            s = rs.uniform(3.0, 6.0) * zz / focal(S)
            sc.append((s, 0.6 * s, 2e-8) if j else (s, 0.8 * s, 0.5 * s))
    P = len(xyz)
    g = make_inputs(xyz, sc, random_quats(P, rs), rs.uniform(0.4, 0.95, P), shs_for(rs.uniform(0, 1, (P, 3)), rs))
    z = g["means3D"][:, 2].numpy()
    assert z[0] == NEAR and z[2] == np.nextafter(NEAR, np.float32(1))
    st = raster.preprocess(S, g["means3D"], g["opacities"], shs=g["shs"], scales=g["scales"], rotations=g["rotations"])
    np.testing.assert_array_equal(st.radii > 0, z > NEAR)
    np.testing.assert_array_equal(raster.mark_visible(S, g["means3D"]), z > NEAR)
    return S, g


GUARD_FACTORS = (1 - 1e-3, 1 + 1e-3, 2.0, 10.0)


def guard_band():
    """tx/tz and ty/tz at +-1.3 tan(fov) * (1 -+ 1e-3), 2 and 10: x alone, y alone, both.  Each splat is large enough for its
    footprint (computed with the clamped Jacobian) to reach into the image."""
    S = settings(96, 64)
    rs = np.random.RandomState(2)
    limx, limy = 1.3 * S.tanfovx, 1.3 * S.tanfovy
    xyz, sc, expect = [], [], []
    for axes in ("x", "y", "xy"):
        for k in GUARD_FACTORS:
            for sgn in (-1.0, 1.0):
                z = rs.uniform(1.0, 3.0)
                ux = sgn * k * limx if "x" in axes else rs.uniform(-0.5, 0.5) * S.tanfovx
                uy = sgn * k * limy if "y" in axes else rs.uniform(-0.5, 0.5) * S.tanfovy
                xyz.append((ux * z, uy * z, z))
                off = max(abs(ux) / S.tanfovx * S.image_width, abs(uy) / S.tanfovy * S.image_height) / 2
                s = (off / 2 + 6.0) * z / focal(S)
                sc.append((s, 0.7 * s, 0.5 * s))
                expect.append(("x" in axes and k > 1, "y" in axes and k > 1))
    P = len(xyz)
    g = make_inputs(xyz, sc, random_quats(P, rs), rs.uniform(0.3, 0.8, P), shs_for(rs.uniform(0, 1, (P, 3)), rs))
    m = g["means3D"].numpy()
    f32 = np.float32
    txtz, tytz = m[:, 0] / m[:, 2], m[:, 1] / m[:, 2]
    lx, ly = f32(1.3) * f32(S.tanfovx), f32(1.3) * f32(S.tanfovy)
    np.testing.assert_array_equal((txtz < -lx) | (txtz > lx), [e[0] for e in expect])
    np.testing.assert_array_equal((tytz < -ly) | (tytz > ly), [e[1] for e in expect])
    st = oracle_forward(S, g)
    assert (st.radii > 0).all(), "every guard-band splat must reach the image"
    blended = np.unique(np.concatenate([st.point_list[st.ranges[t, 0]:st.ranges[t, 1]] for t in range(st.ranges.shape[0])]))
    assert blended.size == P
    return S, g


def offscreen():
    """Centres beyond each side and each corner (rect clipping on all four sides), plus one splat whose radius exceeds int32
    (it must cover the whole grid) and one centre so far off-screen that its rect bounds exceed int32 (culled)."""
    S = settings(96, 64)
    rs = np.random.RandomState(3)
    W, H = S.image_width, S.image_height
    d = 20.0
    spots = [(-d, H / 2), (W - 1 + d, H / 2), (W / 2, -d), (W / 2, H - 1 + d),
             (-d, -d), (W - 1 + d, -d), (-d, H - 1 + d), (W - 1 + d, H - 1 + d)]
    xyz, sc = [], []
    for px, py in spots:
        z = rs.uniform(1.0, 2.0)
        x, y = unproject(S, px + rs.uniform(-2, 2), py + rs.uniform(-2, 2), z)
        xyz.append((x, y, z))
        s = 14.0 * z / focal(S)
        sc.append((s, 0.8 * s, 0.6 * s))
    xyz.append((0.01, -0.02, 50.0)); sc.append((1e9, 1e9, 1e9))                # 3 sqrt(lambda) ~ 8e9 px
    xyz.append((1e9, 0.0, 1.0)); sc.append((0.05, 0.05, 0.05))                 # px ~ 1.3e11: (px - r) / 16 > 2^31
    P = len(xyz)
    opac = np.concatenate([rs.uniform(0.5, 0.9, P - 2), [0.3, 0.9]])
    g = make_inputs(xyz, sc, random_quats(P, rs), opac, shs_for(rs.uniform(0, 1, (P, 3)), rs))
    st = raster.preprocess(S, g["means3D"], g["opacities"], shs=g["shs"], scales=g["scales"], rotations=g["rotations"])
    gx, gy = (W + 15) // 16, (H + 15) // 16
    n = len(spots)
    assert (st.radii[:n] > 0).all()
    r = st.radii[:n].astype(np.float64)
    lo = np.floor((st.means2D[:n] - r[:, None]) / 16)
    hi = np.floor((st.means2D[:n] + r[:, None] + 15) / 16)
    assert (lo[:, 0] < 0).any() and (lo[:, 1] < 0).any() and (hi[:, 0] > gx).any() and (hi[:, 1] > gy).any()
    assert st.radii[n] == INT32_MAX and tuple(st.rects[n]) == (0, 0, gx, gy)
    assert st.radii[n + 1] == 0 and float(st.means2D[n + 1, 0]) == 0.0
    return S, g


def screen_filling():
    """P = 40 splats that each touch all 40 tiles: N = P * T, every list crosses the 32-splat round, and every rect is at least
    32 tiles (the warp-cooperative duplicate emission)."""
    S = settings(128, 80)
    rs = np.random.RandomState(4)
    P = 40
    xyz, sc = [], []
    for i in range(P):
        z = rs.uniform(1.0, 4.0)
        x, y = unproject(S, rs.uniform(40, 88), rs.uniform(25, 55), z)
        xyz.append((x, y, z))
        s = rs.uniform(45.0, 70.0) * z / focal(S)
        sc.append((s, rs.uniform(0.6, 1.0) * s, rs.uniform(0.3, 1.0) * s))
    g = make_inputs(xyz, sc, random_quats(P, rs), rs.uniform(0.04, 0.1, P), shs_for(rs.uniform(0, 1, (P, 3)), rs))
    st = oracle_forward(S, g)
    T = st.ranges.shape[0]
    assert T >= 32 and st.N == P * T and (st.tiles_touched == T).all()
    assert (st.n_contrib > 32).mean() > 0.5, "lists must be blended past the first 32-splat round"
    return S, g


@functools.lru_cache(maxsize=None)
def sliver_sweep(W=256, H=160):
    """Edge-on slivers for the composite kernels' quad cull: major sigma 500 / 1500 / 3000 / 6000 px, 24 orientations, a flat
    (2e-8) or zero minor axis, centred on screen or 0.5-2.5 sigma off-screen along the major axis (the image then sees the
    splat where the terms of the quadratic form are largest).  One splat per scene, so no other splat can hide a pixel the
    cull wrongly skips.  Returns [(tag, Settings, inputs)]; asserts that some blending pixel has a term magnitude
    S = 0.5 (|cx| dx^2 + |cz| dy^2) + |cy dx dy| >= 1e6."""
    S = settings(W, H, sh_degree=0, bg=(0.0, 0.0, 0.0))
    rs = np.random.RandomState(5)
    z = 2.0
    out, smax = [], {}
    for sigma in SLIVER_SIGMAS:
        for minor in SLIVER_MINORS:
            for where in ("on", "off"):
                for k in range(24):
                    th = math.pi * (k + 0.31) / 24
                    u = (math.cos(th), math.sin(th))
                    if where == "on":
                        px, py = W / 2 + rs.uniform(-30, 30), H / 2 + rs.uniform(-20, 20)
                    else:
                        dist = sigma * (0.5 + 0.5 * (k % 5))
                        px, py = W / 2 - dist * u[0] + rs.uniform(-3, 3), H / 2 - dist * u[1] + rs.uniform(-3, 3)
                    x, y = unproject(S, px, py, z)
                    g = make_inputs([(x, y, z)], [(sigma * z / focal(S), minor, 2e-8)], [z_quat(th)], [0.9],
                                    shs_for([[0.8, 0.5, 0.2]], rs, rest=0.0))
                    out.append((f"sigma{sigma}-minor{minor:g}-{where}-{k}", S, g))
                    st = oracle_forward(S, g)
                    s = blend_term_magnitude(st)
                    smax[sigma] = max(smax.get(sigma, 0.0), s)
    assert max(smax.values()) >= 1e6, smax
    sliver_sweep.smax = smax
    return out


def blend_term_magnitude(st):
    """Largest S = 0.5 (|cx| dx^2 + |cz| dy^2) + |cy dx dy| over the pixels where the (single) splat blends, float64."""
    hit = st.n_contrib > 0
    if not hit.any() or not (st.radii > 0).any():
        return 0.0
    i = int(np.flatnonzero(st.radii > 0)[0])
    ys, xs = np.nonzero(hit)
    dx = np.float32(st.means2D[i, 0]) - xs.astype(np.float32)
    dy = np.float32(st.means2D[i, 1]) - ys.astype(np.float32)
    cx, cy, cz = (abs(float(v)) for v in st.conic_opacity[i, :3])
    dx, dy = dx.astype(np.float64), dy.astype(np.float64)
    return float((0.5 * (cx * dx * dx + cz * dy * dy) + cy * np.abs(dx * dy)).max())


def antialiasing():
    """Antialiasing on: tiny splats with det_cov / det 1% below and 1% above the 2.5e-5 floor, centred exactly on pixel centres
    with opacity 0.99 (so they blend their own pixel), among ordinary splats far above the floor."""
    S = settings(64, 48, antialiasing=True)
    rs = np.random.RandomState(6)
    xyz, sc, q, op, ratio = [], [], [], [], []
    for i, fac in enumerate((0.99, 0.99, 0.99, 1.01, 1.01, 1.01)):
        z = 1.0 + 0.25 * i
        r = AA_FLOOR * fac
        a = 0.3 * math.sqrt(r) / (1 - math.sqrt(r))            # raw variance with (a / (a + 0.3))^2 = r
        px, py = 6.0 + 10 * i, 8.0 + 4 * (i % 3)
        xyz.append(snap(S, px, py, z))
        sc.append((math.sqrt(a) * z / focal(S),) * 2 + (0.0,))
        q.append(z_quat(rs.uniform(0, math.pi)))
        op.append(0.99)
        ratio.append(r)
    for i in range(14):
        z = rs.uniform(1.0, 3.0)
        x, y = unproject(S, rs.uniform(0, 64), rs.uniform(0, 48), z)
        xyz.append((x, y, z))
        s = rs.uniform(1.0, 5.0) * z / focal(S)
        sc.append((s, rs.uniform(0.2, 1.0) * s, rs.uniform(0.0, 1.0) * s))
        q.append(random_quats(1, rs)[0])
        op.append(rs.uniform(0.3, 0.9))
    P = len(xyz)
    g = make_inputs(xyz, sc, q, op, shs_for(rs.uniform(0, 1, (P, 3)), rs))
    st = oracle_forward(S, g)
    h = st.conic_opacity[:6, 3] / g["opacities"][:6, 0].numpy()
    floor = np.float32(math.sqrt(AA_FLOOR))
    assert (np.abs(h[:3] - floor) <= 1e-6 * floor).all(), h        # clamped at the floor
    assert (h[3:] > floor * (1 + 2e-3)).all(), h                     # just above it
    assert (st.n_contrib > 0).sum() > 100
    for i in range(6):          # each tiny splat blends at least its own pixel
        px, py = int(st.means2D[i, 0]), int(st.means2D[i, 1])
        assert st.means2D[i, 0] == px and st.means2D[i, 1] == py and st.n_contrib[py, px] > 0
    return S, g


SH_AXES = {"+x": (1, 0, 0), "-x": (-1, 0, 0), "+y": (0, 1, 0), "-y": (0, -1, 0), "+z": (0, 0, 1), "-z": (0, 0, -1)}


def sh_case(degree, axis):
    """SH degree `degree`, camera looking along `axis`: the splats sit on and around the optical axis, so their view
    directions are (nearly) +-x, +-y or +-z, and their colours have zero, one, two or three channels below 0 (clamped)."""
    eye = np.array([0.3, -0.2, 0.1])
    a = np.asarray(SH_AXES[axis], np.float64)
    cam = scenes.look_at_camera(tuple(eye), tuple(eye + a), 40, 32)
    S = settings_from_camera(cam, sh_degree=degree, bg=(0.1, 0.4, 0.8))
    rs = np.random.RandomState(7 + degree * 10 + list(SH_AXES).index(axis))
    R = cam.world_view_transform.numpy()[:3, :3]          # transposed storage: rows of R^T are the camera axes
    right, down = R[:, 0], R[:, 1]
    P = 12
    xyz = []
    for i in range(P):
        o = (0.0, 0.0) if i == 0 else rs.uniform(-0.25, 0.25, 2)
        xyz.append(eye + 1.5 * a + o[0] * right + o[1] * down)
    rgb = rs.uniform(0.3, 0.9, (P, 3))
    for i in range(P):
        neg = rs.permutation(3)[: i % 4]
        rgb[i, neg] = -rs.uniform(0.4, 0.8, len(neg))
    s = rs.uniform(0.02, 0.06, (P, 1)) * np.array([1.0, 0.7, 0.5])
    g = make_inputs(xyz, s, random_quats(P, rs), rs.uniform(0.4, 0.9, P), shs_for(rgb, rs, rest=0.04))
    st = raster.preprocess(S, g["means3D"], g["opacities"], shs=g["shs"], scales=g["scales"], rotations=g["rotations"])
    assert (st.radii > 0).all()
    assert {1, 2, 3} <= set(st.clamped.sum(1).tolist())
    return S, g


def opacity_edges():
    """Opacity 1 exactly on a pixel centre (alpha clamped at 0.99), opacity below 1/255 (tau = -1: never blends) and exactly
    float32(1/255) on a pixel centre (alpha == 1/255 there: blends, and the pixel is threshold-ambiguous)."""
    S = settings(48, 32)
    rs = np.random.RandomState(8)
    z = 1.5
    spots = [(10.0, 10.0, 1.0), (30.0, 12.0, 0.003), (20.0, 24.0, float(np.float32(1.0 / 255.0)))]
    xyz = [snap(S, px, py, z) for px, py, _ in spots]
    op = [o for *_, o in spots]
    sc = [(3.0 * z / focal(S), 2.0 * z / focal(S), 1e-3)] * 3
    for i in range(6):
        zz = rs.uniform(2.0, 3.0)
        x, y = unproject(S, rs.uniform(0, 48), rs.uniform(0, 32), zz)
        xyz.append((x, y, zz))
        s = rs.uniform(2.0, 5.0) * zz / focal(S)
        sc.append((s, 0.7 * s, 0.4 * s))
        op.append(rs.uniform(0.3, 0.8))
    P = len(xyz)
    q = np.concatenate([np.tile([[1.0, 0, 0, 0]], (3, 1)), random_quats(P - 3, rs)])
    g = make_inputs(xyz, sc, q, op, shs_for(rs.uniform(0, 1, (P, 3)), rs))
    st = oracle_forward(S, g)
    for i, (px, py, _) in enumerate(spots):
        assert st.means2D[i, 0] == px and st.means2D[i, 1] == py
    assert st.conic_opacity[0, 3] == 1.0 and 0 < st.conic_opacity[1, 3] < 1.0 / 255.0
    assert st.conic_opacity[2, 3] == np.float32(1.0 / 255.0)
    assert abs(float(st.final_T[10, 10]) - 0.01) < 1e-6, "opacity 1 at the pixel centre must blend at alpha 0.99"
    assert st.ambiguous[24, 20] == 1 and st.n_contrib[24, 20] > 0
    return S, g


EXACT_SPOTS = [(0.0, 0.0), (7.0, 3.0), (7.5, 9.0), (8.0, 15.5), (15.0, 16.0), (15.5, 7.5), (16.0, 24.0), (23.5, 31.0),
               (31.0, 8.0), (32.0, 23.5), (40.0, 16.0), (63.0, 31.0)]


def exact_positions():
    """Centres exactly on pixel centres (power exactly 0 there) and on quad / tile borders (x or y = 7, 7.5, 8, 15, 15.5, 16,
    ...), so the cull's inside test and its edge minimisation both meet their boundaries.  64 x 32: (2 px + 1) / W is then
    dyadic, so every pixel centre is reachable exactly."""
    S = settings(64, 32)
    rs = np.random.RandomState(9)
    xyz, sc = [], []
    for i, (px, py) in enumerate(EXACT_SPOTS):
        z = 1.0 + 0.1 * i
        xyz.append(snap(S, px, py, z))
        s = rs.uniform(1.5, 4.0) * z / focal(S)
        sc.append((s, rs.uniform(0.1, 1.0) * s, rs.uniform(0.1, 1.0) * s))
    P = len(xyz)
    g = make_inputs(xyz, sc, random_quats(P, rs), rs.uniform(0.3, 0.9, P), shs_for(rs.uniform(0, 1, (P, 3)), rs))
    st = oracle_forward(S, g)
    np.testing.assert_array_equal(st.means2D, np.float32(EXACT_SPOTS))
    return S, g


def depth_ties():
    """Overlapping splats at one identical fp32 depth (two of them identical in every parameter): the sort's tie order."""
    S = settings(48, 32)
    rs = np.random.RandomState(10)
    P = 8
    z = 1.7
    xyz, sc = [], []
    for i in range(P):
        x, y = unproject(S, 24 + rs.uniform(-6, 6), 16 + rs.uniform(-5, 5), z)
        xyz.append((x, y, z))
        s = rs.uniform(3.0, 6.0) * z / focal(S)
        sc.append((s, 0.8 * s, 0.5 * s))
    q = random_quats(P, rs)
    op = rs.uniform(0.3, 0.7, P)
    shs = shs_for(rs.uniform(0, 1, (P, 3)), rs)
    xyz[5], sc[5], q[5], op[5] = xyz[4], sc[4], q[4], op[4]
    g = make_inputs(xyz, sc, q, op, shs)
    st = oracle_forward(S, g)
    assert np.unique(st.depths).size == 1 and (st.radii > 0).all()
    return S, g


def ragged(W=93, H=61):
    """W and H multiples of neither 8 nor 16 (partial quads and tiles), an ordinary random scene."""
    cam = scenes.look_at_camera((2.6, 0.4, 1.2), (0, 0, 0), W, H)
    S = settings_from_camera(cam, bg=(0.2, 0.5, 0.9))
    g = random_gaussians(150, seed=11, extent=0.8, scale_mu=-2.4)
    assert W % 8 and H % 8
    return S, g


# name -> builder of the scenes that are small enough for the dense float64 model (P <= ~300, images <= ~128x80), with the
# tolerances the dense comparison holds them to: forward abs per pixel, gradients max err / max |ref|
CASES = {
    "near_plane": near_plane,
    "guard_band": guard_band,
    "offscreen": offscreen,
    "screen_filling": screen_filling,
    "antialiasing": antialiasing,
    "opacity_edges": opacity_edges,
    "exact_positions": exact_positions,
    "depth_ties": depth_ties,
    "ragged": ragged,
    "ragged_small": functools.partial(ragged, 37, 21),
}
for _d in range(4):
    for _a in SH_AXES:
        CASES[f"sh{_d}{_a}"] = functools.partial(sh_case, _d, _a)
