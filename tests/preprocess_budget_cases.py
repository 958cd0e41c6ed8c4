"""Scenes and the per-element check of the preprocess backward against its float64 reference (oracle/preprocess64.py).

Every builder returns (Settings, inputs) for the CPU tests (tests/test_preprocess_budget.py) and the GPU tests
(tests/test_gpu_preprocess_budget.py); `record` makes the per-Gaussian [P,10] record the preprocess backward reads, from
the C oracle's composite backward under random upstream gradients."""
from __future__ import annotations

import functools
import math

import numpy as np
import torch

import raster_edge_cases as rec
from gms_b200 import scenes
from helpers import random_gaussians, settings_from_camera
from oracle import preprocess64, raster

# gradient name of the rasterizer's autograd outputs -> key of raster.preprocess_backward / preprocess_backward64
GRAD_KEYS = {"means3D": "dL_dmeans3D", "means2D": "dL_dmeans2D", "opacities": "dL_dopacity", "shs": "dL_dsh",
             "colors_precomp": "dL_dcolors_precomp", "scales": "dL_dscales", "rotations": "dL_drotations",
             "cov3D_precomp": "dL_dcov3D", "colors_sh": "dL_dcolors_sh"}


def _cam(W=160, H=112, eye=(2.2, 1.5, 0.9), **kw):
    return settings_from_camera(scenes.look_at_camera(eye, (0, 0, 0), W, H), **kw)


def _random(P, seed, **kw):
    return _cam(**kw), random_gaussians(P, seed=seed, extent=1.2, scale_mu=-2.4)


def flat(edge_on):
    """Flat Gaussians (s0 = 2e-8) facing the camera (flat axis along the view axis) or seen edge-on (flat axis across it)."""
    S = rec.settings(96, 64)
    rs = np.random.RandomState(21 + edge_on)
    P = 24
    xyz, sc, q = [], [], []
    for _ in range(P):
        z = rs.uniform(1.0, 3.0)
        x, y = rec.unproject(S, rs.uniform(8, 88), rs.uniform(8, 56), z)
        xyz.append((x, y, z))
        s = rs.uniform(2.0, 8.0) * z / rec.focal(S)
        sc.append((2e-8, s, rs.uniform(0.3, 1.0) * s))
        th = rs.uniform(0, math.pi)     # flat axis = R's first column: about y by 90 deg puts it along z (face-on)
        qy = np.array([math.cos(math.pi / 4), 0, math.sin(math.pi / 4), 0]) if not edge_on else np.array([1.0, 0, 0, 0])
        qz = rec.z_quat(th)
        q.append(_qmul(qz, qy))
    g = rec.make_inputs(xyz, sc, q, rs.uniform(0.4, 0.9, P), rec.shs_for(rs.uniform(0, 1, (P, 3)), rs))
    return S, g


def _qmul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def unnormalised(norm):
    """Quaternions of norm 0.5 or 2: the upstream rotation formula does not normalise them."""
    S, g = _random(300, 23)
    g["rotations"] = g["rotations"] * norm
    return S, g


def scale_modifier():
    return _cam(scale_modifier=0.7), random_gaussians(300, seed=24, extent=1.2, scale_mu=-2.2)


def precomputed():
    """colors_precomp and cov3D_precomp instead of SH and scale / rotation (the covariance of a first forward)."""
    S, g = _random(300, 25)
    st = raster.preprocess(S, g["means3D"], g["opacities"], shs=g["shs"], scales=g["scales"], rotations=g["rotations"])
    rs = np.random.RandomState(25)
    return S, dict(means3D=g["means3D"], opacities=g["opacities"], colors_precomp=torch.tensor(rs.uniform(0, 1, (300, 3)), dtype=torch.float32),
                   cov3D_precomp=torch.tensor(st.cov3Ds))


def sh_width(M):
    """M SH coefficients per Gaussian and the degree they hold (M = 1, 4, 9: the narrow-row paths)."""
    S, g = _random(300, 26, sh_degree=int(round(math.sqrt(M))) - 1)
    g["shs"] = g["shs"][:, :M].contiguous()
    return S, g


def sh_degree(d):
    """M = 16 rows with active degree d."""
    return _random(300, 27 + d, sh_degree=d)


def count(P):
    """P = 1, 31 (partial warp), 4099 (partial block and warp of the staged tiles)."""
    S, g = _random(P, 28, W=192, H=128)
    g["means3D"] = g["means3D"] * (0.3 if P == 1 else 1.0)
    return S, g


def aa_random():
    return _random(600, 29, antialiasing=True)


def sh_case_all():
    """sh_case for every degree and view axis merged: view directions along each axis, colours clamped in 0-3 channels."""
    return [(f"sh{d}{a}", functools.partial(rec.sh_case, d, a)) for d in range(4) for a in rec.SH_AXES]


SCENES = {
    "near_plane": rec.near_plane, "guard_band": rec.guard_band, "antialiasing": rec.antialiasing,
    "screen_filling": rec.screen_filling, "offscreen": rec.offscreen,
    "flat_face_on": functools.partial(flat, False), "flat_edge_on": functools.partial(flat, True),
    "quat_half": functools.partial(unnormalised, 0.5), "quat_two": functools.partial(unnormalised, 2.0),
    "scale_modifier": scale_modifier, "precomputed": precomputed, "aa_random": aa_random,
    **{f"M{m}": functools.partial(sh_width, m) for m in (1, 4, 9)},
    **{f"deg{d}": functools.partial(sh_degree, d) for d in range(4)},
    **{f"P{p}": functools.partial(count, p) for p in (1, 31, 4099)},
    **dict(sh_case_all()),
}


def forward(S, g):
    return raster.forward(S, g["means3D"], g["opacities"], shs=g.get("shs"), colors_precomp=g.get("colors_precomp"),
                          scales=g.get("scales"), rotations=g.get("rotations"), cov3D_precomp=g.get("cov3D_precomp"))


def upstream(S, seed=1):
    rs = np.random.RandomState(seed)
    H, W = S.image_height, S.image_width
    return rs.randn(3, H, W).astype(np.float32), rs.randn(H, W).astype(np.float32)


def record(st, dL_dcolor, dL_dinv):
    """The C oracle's composite backward as the fp32 [P,10] record (mean2D, conic, opacity, rgb, inverse depth)."""
    c = raster.composite_backward(st, dL_dcolor, dL_dinv)
    return np.ascontiguousarray(np.concatenate([c["dL_dmean2D"], c["dL_dconic"], c["dL_dopacity"][:, None], c["dL_dcolor"],
                                                c["dL_dinvdepth"][:, None]], 1), np.float32)


def budget_ratios(got, ref64, budget):
    """|got - ref64| / budget elementwise (0 where equal, inf where the budget is 0 and they differ, NaN for NaN)."""
    got = np.asarray(got, np.float64).reshape(ref64.shape)
    err = np.abs(got - ref64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(err == 0, 0.0, err / budget)


def check_per_element(got, r, vis=None):
    """{gradient name: worst ratio} over the gradients in `got` (keyed like the rasterizer's autograd outputs); rows not in
    `vis` (if given) are skipped."""
    worst = {}
    for kg, arr in got.items():
        kr = GRAD_KEYS.get(kg)
        if kr is None or kr not in r["ref64"] or arr is None:
            continue
        ratio = budget_ratios(arr, r["ref64"][kr], r["budget"][kr])
        if vis is not None:
            ratio = ratio[vis]
        worst[kg] = float(np.nan_to_num(ratio, nan=np.inf).max()) if ratio.size else 0.0
    return worst


def assert_preprocess_per_element(st, got, dgeom, label="", r=None):
    """Every element of the preprocess backward's outputs in `got` within its budget around the float64 reference evaluated on
    the same record `dgeom`; a Gaussian with budget 0 (culled, or a zero record) must come out exactly 0.  Prints the worst
    ratio per gradient."""
    r = preprocess64.preprocess_backward64(st, dgeom) if r is None else r
    for k, v in r["budget"].items():
        assert np.isfinite(v).all() and np.isfinite(r["ref64"][k]).all(), f"non-finite float64 reference or budget for {k}"
    for kg, arr in got.items():
        if GRAD_KEYS.get(kg) in r["ref64"]:
            assert np.isfinite(arr).all(), f"non-finite preprocess backward {kg}"
    worst = check_per_element(got, r)
    print(f"[per-element{(' ' + label) if label else ''}] worst |gpu - ref64| / budget: "
          + ", ".join(f"{k} {w:.3g}" for k, w in worst.items()) + f"; {int(r['ambiguous'].sum())} branch-ambiguous Gaussians")
    for kg, w in worst.items():
        if not w <= 1.0:
            kr = GRAD_KEYS[kg]
            ratio = budget_ratios(got[kg], r["ref64"][kr], r["budget"][kr])
            idx = np.unravel_index(int(np.argmax(np.nan_to_num(ratio, nan=np.inf))), ratio.shape)
            got_v = float(np.asarray(got[kg], np.float64).reshape(ratio.shape)[idx])
            raise AssertionError(f"preprocess backward {kg} outside its budget at {int((~(ratio <= 1)).sum())} elements, e.g. {idx}: "
                                 f"got {got_v:.9g} ref64 {r['ref64'][kr][idx]:.9g} budget {r['budget'][kr][idx]:.3g}")
    return worst
