"""Run the product (CUDA, through the Python shim -> C ABI) and the oracle on the same inputs."""
import numpy as np
import torch

import diff_gaussian_rasterization as dgr
from gms_b200 import rasterizer
from oracle import expansion as oexp
from oracle import raster
from preprocess_budget_cases import assert_preprocess_per_element


def gpu_settings(S: raster.Settings, dev="cuda"):
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=dev)
    return dgr.GaussianRasterizationSettings(
        image_height=S.image_height, image_width=S.image_width, tanfovx=S.tanfovx, tanfovy=S.tanfovy, bg=t(S.bg),
        scale_modifier=S.scale_modifier, viewmatrix=t(S.viewmatrix), projmatrix=t(S.projmatrix), sh_degree=S.sh_degree,
        campos=t(S.campos), prefiltered=False, debug=False, antialiasing=S.antialiasing)


def run_gpu(S, inputs, dL_dcolor=None, dL_dinv=None, dev="cuda"):
    """inputs: dict of CPU tensors (means3D, opacities, shs|colors_precomp, scales+rotations|cov3D_precomp).
    Returns (color, radii, invdepth, debug-state dict, grads dict or None)."""
    rasterizer.KEEP_DEBUG = True
    rs = gpu_settings(S, dev)
    t = {k: v.to(dev).float().clone().requires_grad_(dL_dcolor is not None) for k, v in inputs.items() if v is not None}
    P = t["means3D"].shape[0]
    m2d = torch.zeros(P, 3, device=dev, requires_grad=dL_dcolor is not None)
    r = dgr.GaussianRasterizer(raster_settings=rs)
    color, radii, invd = r(means3D=t["means3D"], means2D=m2d, opacities=t["opacities"], shs=t.get("shs"),
                           colors_precomp=t.get("colors_precomp"), scales=t.get("scales"), rotations=t.get("rotations"),
                           cov3D_precomp=t.get("cov3D_precomp"))
    dbg = rasterizer.last_debug
    state = rasterizer.forward_debug_state(dbg["scratch"], dbg["num_rendered"], P, S.image_width, S.image_height, radii)
    state["num_rendered"] = dbg["num_rendered"]
    grads = None
    if dL_dcolor is not None:
        loss = (color * torch.tensor(dL_dcolor, device=dev)).sum()
        if dL_dinv is not None:
            loss = loss + (invd[0] * torch.tensor(dL_dinv, device=dev)).sum()
        loss.backward()
        grads = {k: v.grad.detach().cpu().numpy() for k, v in t.items() if v.grad is not None}
        grads["means2D"] = m2d.grad.detach().cpu().numpy()
        # what the composite backward handed to the preprocess backward (debug view of the per-Gaussian accumulators)
        after = rasterizer.forward_debug_state(dbg["scratch"], dbg["num_rendered"], P, S.image_width, S.image_height, radii,
                                               bin_state=dbg.get("bin_state"))
        if "dgeom" in after:
            grads["_dgeom"] = after["dgeom"].cpu().numpy()
    torch.cuda.synchronize()
    return color.detach().cpu().numpy(), radii.cpu().numpy(), invd.detach().cpu().numpy(), \
        {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in state.items()}, grads


def run_oracle(S, inputs, dL_dcolor=None, dL_dinv=None):
    st = raster.forward(S, inputs["means3D"], inputs["opacities"], shs=inputs.get("shs"),
                        colors_precomp=inputs.get("colors_precomp"), scales=inputs.get("scales"),
                        rotations=inputs.get("rotations"), cov3D_precomp=inputs.get("cov3D_precomp"))
    g = None
    if dL_dcolor is not None:
        g = raster.backward(st, dL_dcolor, dL_dinv)
    return st, g


# gradients of the raw mesh-Gaussian parameters (oracle_chain) against the oracle, as max err / max |ref|; 2e-4 for the others
GRAD_TOL = {"vertices": 5e-3, "_scale": 5e-3, "_alpha": 1e-3}     # through the near-singular 2D covariance (DESIGN.md 2.2)


def oracle_chain(p, S, dC, gpu, triangles=None):
    """Oracle image and gradients of sum(image * dC) w.r.t. the raw mesh-Gaussian parameters.  `gpu` = the (means3D,
    scales, rotations) the GPU run handed to the rasterizer: they must agree with the oracle's expansion to fp32 rounding
    and are what the oracle rasterizes (so that integer outputs can be compared bit for bit); the gradient chain runs
    through the oracle's own expansion graph."""
    tv, ta, ts = (x.clone().requires_grad_(True) for x in (p.vertices, p._alpha, p._scale))
    if triangles is None:
        xyz, sl, rr, _, _ = oexp.expand(tv, p.faces, ta, ts)
    else:
        alpha, _, _ = oexp.update_alpha(ta, tv, p.faces)
        xyz = torch.matmul(alpha, triangles).reshape(-1, 3)
        sl, rr = oexp.prepare_scaling_rot(triangles, ts, ta.shape[1])
    top = p._opacity.clone().requires_grad_(True)
    sc, rot, op, fe = oexp.activate(sl, rr, top, p._features_dc, p._features_rest)
    gx, gs, gr = (t.detach().cpu() for t in gpu)
    assert float((gx - xyz.detach()).abs().max()) <= 2e-6 and float((gr - rot.detach()).abs().max()) <= 4e-6
    assert float(((gs - sc.detach()).abs() / sc.detach()).max()) <= 1e-5
    st = raster.forward(S, gx, op.detach(), shs=fe.contiguous(), scales=gs, rotations=gr)
    g = raster.backward(st, dC)
    outs = [(xyz, g["dL_dmeans3D"]), (sc, g["dL_dscales"]), (rot, g["dL_drotations"]), (op, g["dL_dopacity"])]
    outs = [(t, torch.tensor(gr).reshape(t.shape)) for t, gr in outs if t.requires_grad]     # animated path: rotation is a constant of the triangles
    torch.autograd.backward([t for t, _ in outs], [gr for _, gr in outs])
    grads = dict(vertices=tv.grad, _alpha=ta.grad, _scale=ts.grad, _opacity=top.grad,
                 _features_dc=torch.tensor(g["dL_dsh"][:, :1]), _features_rest=torch.tensor(g["dL_dsh"][:, 1:]))
    return st, grads


def assert_forward_parity(st, color, radii, invd, state, tol=1e-5, max_ambiguous=5e-4):
    """Bit-exact indices, <= tol per pixel (threshold-ambiguous pixels get a bounded looser check; at most `max_ambiguous` of
    the image may be threshold-ambiguous)."""
    np.testing.assert_array_equal(radii, st.radii)
    assert state["num_rendered"] == st.N
    if st.radii.shape[0]:
        np.testing.assert_array_equal(state["tiles_touched"].astype(np.uint32), st.tiles_touched)
        vis = st.radii > 0
        np.testing.assert_array_equal(state["means2D"].view(np.uint32)[vis], st.means2D.view(np.uint32)[vis])
        np.testing.assert_array_equal(state["depths"].view(np.uint32)[vis], st.depths.view(np.uint32)[vis])
        np.testing.assert_array_equal(state["conic_opacity"].view(np.uint32)[vis], st.conic_opacity.view(np.uint32)[vis])
        np.testing.assert_array_equal(state["cov3D"].view(np.uint32)[vis], st.cov3Ds.view(np.uint32)[vis])
        np.testing.assert_array_equal(state["clamped"][vis], st.clamped[vis])
        np.testing.assert_allclose(state["rgb"][vis], st.rgb[vis], rtol=1e-6, atol=1e-6)
    np.testing.assert_array_equal(state["point_list"].astype(np.uint32), st.point_list)
    np.testing.assert_array_equal(state["tile_keys"].astype(np.uint64), st.keys_sorted >> np.uint64(32))
    np.testing.assert_array_equal(state["ranges"], st.ranges)
    ok = assert_image_parity(st, color, tol, max_ambiguous)
    np.testing.assert_array_equal(state["n_contrib"][ok], st.n_contrib[ok])
    assert np.abs(invd - st.invdepth)[:, ok].max() <= tol
    assert np.abs(state["final_T"] - st.final_T)[ok].max() <= tol


def assert_image_parity(st, color, tol=1e-5, max_ambiguous=5e-4):
    """<= tol per pixel outside the threshold-ambiguous pixels; returns the mask of those other pixels.
    Threshold-ambiguous pixels: the oracle flags a pixel when one of its skip / stop decisions (alpha < 1/255,
    T(1-alpha) < 1e-4) lies within the +-1e-6 relative band in which exp() (GPU: ex2.approx.ftz) may fall on the other side.
    They are REPORTED (count, worst error) and bounded by the largest change one flipped decision can cause: a splat
    blended at alpha = 1/255 with unit transmittance moves a channel by <= |c - behind| / 255 <= max colour / 255."""
    ok = st.ambiguous == 0
    n_amb = int((~ok).sum())
    err = np.abs(color - st.color)
    err_ok = float(err[:, ok].max()) if ok.any() else 0.0
    err_amb = float(err[:, ~ok].max()) if n_amb else 0.0
    cmax = float(max(1.0, np.abs(st.rgb).max())) if st.radii.shape[0] else 1.0
    print(f"[parity] {st.settings.image_width}x{st.settings.image_height} P={st.radii.shape[0]} N={st.N}: max|image-oracle| = {err_ok:.2e}; "
          f"threshold-ambiguous pixels = {n_amb} ({n_amb / ok.size:.1e} of the image), worst there = {err_amb:.2e} (bound {cmax / 255:.1e})")
    assert n_amb <= max(4, max_ambiguous * ok.size), f"too many threshold-ambiguous pixels: {n_amb}"
    assert err_ok <= tol, err_ok
    assert err_amb <= 2.0 * cmax / 255.0, err_amb
    return ok


# Gradients w.r.t. scales / rotations / cov3D go through the inverse of a nearly singular 2D covariance (flat mesh
# Gaussians, s0 ~ 2e-8): the summation-order noise of the fp32 atomics in dL/dconic is amplified by that Jacobian (the stock
# extension has the same non-determinism; the oracle sums in double).  The backward pass is therefore checked in its TWO
# LINEAR STAGES, each at a conditioning-independent tolerance (assert_backward_stages):
#   (1) composite backward:  GPU per-Gaussian sums `dgeom`  vs  oracle composite_backward (double accumulation)
#   (2) preprocess backward: GPU parameter gradients        vs  oracle preprocess_backward fed THE GPU's dgeom
# (1) and (2) together imply the end-to-end gradient up to |J| * err(1); the end-to-end comparison below is kept as a sanity
# check with the measured amplification as its slack.
ILL_CONDITIONED = {"scales": 25.0, "rotations": 25.0, "cov3D_precomp": 25.0, "means3D": 2.5}


# Stage 2 evaluates ONE formula per Gaussian in fp32 on both sides (GPU: nvcc contracts a*b+c into FMAs; oracle: gcc
# -ffp-contract=off): for means3D / opacity / SH the two agree to ~1e-7.  The scale / rotation / cov3D gradients go through
# dL/dM = 2 M dL/dSigma of a nearly singular Sigma (flat mesh Gaussians, s0 ~ 1e-8): the contraction alone moves them by up to
# 2e-3 of max (measured: config 4, 1080p), with identical inputs -- that is the conditioning of the formula, not of the kernel.
STAGE2_TOL = {"scales": 5e-3, "rotations": 5e-3, "cov3D_precomp": 5e-3, "means3D": 5e-4}   # means3D: the J*W chain of near-edge-on splats, measured <= 9e-5


COMPOSITE_GROUPS = {"dL_dmean2D": slice(0, 2), "dL_dconic": slice(2, 5), "dL_dopacity": slice(5, 6), "dL_dcolor": slice(6, 9),
                    "dL_dinvdepth": slice(9, 10)}
COMPONENTS = ("mean2D.x", "mean2D.y", "conic.xx", "conic.xy", "conic.yy", "opacity", "rgb.r", "rgb.g", "rgb.b", "invdepth")


def composite_floor_errors(st, dg, comp):
    """The global stage-1 measure: per group, max over the visible Gaussians of |gpu - oracle| / max |oracle|."""
    vis = st.radii > 0
    out = {}
    for k, sl in COMPOSITE_GROUPS.items():
        got = dg[:, sl].astype(np.float64)
        ref = np.asarray(comp[k], np.float64).reshape(got.shape)
        scale = max(np.abs(ref).max(), 1e-30)
        out[k] = float(np.abs(got - ref)[vis].max() / scale) if vis.any() else 0.0
    return out


def composite_budget_ratios(dg, ref64, budget):
    """|gpu - ref64| / budget per Gaussian and component (0 where both are exactly equal, inf where the budget is 0 and the
    value is not, NaN where the value is NaN)."""
    err = np.abs(np.asarray(dg, np.float64)[:, :10] - ref64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(err == 0, 0.0, err / budget)


# Gaussians whose budget is mostly the allowance of threshold-ambiguous pixels (amb_share > 0.5), as a share of those with any
# gradient: measured <= 6.5 % on the random parity scenes, whose few ambiguous pixels are mostly the T < 1e-4 stop deep in a
# list; 10 % keeps the allowance from quietly taking over a scene.
AMB_MOSTLY_MAX = 0.10


def assert_composite_per_gaussian(st, dgeom, ref64, budget, amb_share=None, label=""):
    """Every Gaussian and every component of the composite backward's per-Gaussian record: |gpu - ref64| <= budget, the float64
    reference and the a-priori budget of oracle.raster.composite_backward64.  A Gaussian that blends nowhere has budget 0
    and must come out exactly zero.  Prints the worst ratio per component."""
    assert np.isfinite(ref64).all() and np.isfinite(budget).all(), "non-finite float64 reference or budget"
    finite = np.isfinite(np.asarray(dgeom)[:, :10])
    assert finite.all(), f"non-finite composite backward at {int((~finite).sum())} elements, e.g. {np.argwhere(~finite)[0].tolist()}"
    r = composite_budget_ratios(dgeom, ref64, budget)
    worst = r.max(0) if r.shape[0] else np.zeros(10)
    has = (budget > 0).any(1)
    mostly = int((amb_share > 0.5).sum()) if amb_share is not None else 0
    print(f"[per-Gaussian{(' ' + label) if label else ''}] worst |gpu - ref64| / budget: "
          + ", ".join(f"{c} {w:.3g}" for c, w in zip(COMPONENTS, worst))
          + f"; {int(has.sum())} Gaussians with a gradient, {mostly} of them mostly ambiguous-pixel allowance")
    bad = np.argwhere(~(r <= 1))
    assert bad.shape[0] == 0, (f"composite backward outside its budget at {bad.shape[0]} elements, e.g. Gaussian {bad[0][0]} "
                               f"{COMPONENTS[bad[0][1]]}: gpu {float(dgeom[bad[0][0], bad[0][1]]):.9g} ref64 "
                               f"{ref64[bad[0][0], bad[0][1]]:.9g} budget {budget[bad[0][0], bad[0][1]]:.3g}")
    assert mostly <= AMB_MOSTLY_MAX * max(int(has.sum()), 1), f"{mostly} of {int(has.sum())} budgets are mostly allowance"
    return worst


def assert_backward_stages(st, g_gpu, g_ref, tol_composite=2e-5, tol_pre=5e-5):
    dg = g_gpu.get("_dgeom")
    comp = g_ref.get("_composite")
    if dg is None or comp is None:
        return False
    msg = []
    for k, e in composite_floor_errors(st, dg, comp).items():
        msg.append(f"{k} {e:.1e}")
        assert e <= tol_composite, f"composite backward {k}: {e:.3e} > {tol_composite}"
    assert "_upstream" in g_ref, "the oracle gradients carry no upstream gradients (_upstream): the per-Gaussian check needs them"
    r = raster.composite_backward64(st, *g_ref["_upstream"])
    assert_composite_per_gaussian(st, dg, r["ref64"], r["budget"], r["amb_share"])
    # stage 2: the oracle's preprocess backward on the GPU's own sums
    fed = dict(dL_dmean2D=dg[:, 0:2].astype(np.float64), dL_dconic=dg[:, 2:5].astype(np.float64), dL_dopacity=dg[:, 5].astype(np.float64),
               dL_dcolor=dg[:, 6:9].astype(np.float64), dL_dinvdepth=dg[:, 9].astype(np.float64))
    ref2 = raster.preprocess_backward(st, fed)
    pairs = [("means3D", "dL_dmeans3D"), ("opacities", "dL_dopacity"), ("shs", "dL_dsh"), ("colors_precomp", "dL_dcolors_precomp"),
             ("scales", "dL_dscales"), ("rotations", "dL_drotations"), ("cov3D_precomp", "dL_dcov3D")]
    for kg, kr in pairs:
        if kg in g_gpu and ref2.get(kr) is not None:
            a, b = g_gpu[kg].astype(np.float64), np.asarray(ref2[kr], np.float64).reshape(g_gpu[kg].shape)
            e = np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)
            msg.append(f"{kg} {e:.1e}")
            assert e <= STAGE2_TOL.get(kg, tol_pre), f"preprocess backward {kg}: {e:.3e} > {STAGE2_TOL.get(kg, tol_pre)}"
    print("[parity] backward stages (max err / max|ref|): " + ", ".join(msg))
    # stage 2 per element: every parameter gradient within its budget around the float64 reference on the GPU's own record
    # (oracle/preprocess64.py); dL/dmeans2D is the record's mean2D, bit for bit
    got = {k: g_gpu[k] for k in ("means3D", "means2D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp")
           if k in g_gpu}
    assert_preprocess_per_element(st, got, dg)
    return True


def assert_grad_parity(g_gpu, g_ref, tol=2e-4, st=None, tol_composite=2e-5):
    pairs = [("means3D", "dL_dmeans3D"), ("means2D", "dL_dmeans2D"), ("opacities", "dL_dopacity"), ("shs", "dL_dsh"),
             ("colors_precomp", "dL_dcolors_precomp"), ("scales", "dL_dscales"), ("rotations", "dL_drotations"),
             ("cov3D_precomp", "dL_dcov3D")]
    checked = 0
    for kg, kr in pairs:
        if kg in g_gpu and g_ref.get(kr) is not None:
            a, b = g_gpu[kg].astype(np.float64), np.asarray(g_ref[kr], np.float64).reshape(g_gpu[kg].shape)
            scale = max(np.abs(b).max(), 1e-20)
            err = np.abs(a - b).max() / scale
            lim = tol * ILL_CONDITIONED.get(kg, 1.0)
            assert err <= lim, f"grad {kg}: max err / max |ref| = {err:.3e} > {lim}"
            checked += 1
    assert checked >= 5
    if st is not None:
        assert_backward_stages(st, g_gpu, g_ref, tol_composite=tol_composite)
