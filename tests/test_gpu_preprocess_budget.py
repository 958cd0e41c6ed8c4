"""The preprocess backward kernel (k_preprocess_bwd) per element: every parameter gradient against the float64 reference of
oracle/preprocess64.py evaluated on the kernel's own per-Gaussian record (the composite backward's `dgeom`), within the
a-priori budget, so that stage 2 is tested apart from any composite noise.  dL/dmeans2D must be the record's mean2D bit
for bit, with a zero third column.

Paths: SH rows per lane, staged through shared memory and processed in place (option "sh_staged" 0 / 1 / 2) under both
launch bounds ("pre_bwd_minblocks" 1 / 4); the factored SH gradient (RasterGrads.dL_dcolors_sh set: the kernel writes the
clamp-masked colour gradient instead of SH rows); the narrow SH rows (M < 16); antialiasing on and off; precomputed colours
and covariances.  The scenes are tests/preprocess_budget_cases.py's."""
import ctypes as C

import numpy as np
import pytest
import torch

import diff_gaussian_rasterization as dgr
import preprocess_budget_cases as pbc
from gms_b200 import _lib, rasterizer
from gpu_helpers import gpu_settings, run_gpu
from oracle import preprocess64

pytestmark = pytest.mark.gpu


def _run(name):
    S, g = pbc.SCENES[name]()
    st = pbc.forward(S, g)
    dC, dD = pbc.upstream(S)
    _, radii, _, state, grads = run_gpu(S, g, dC, dD)
    np.testing.assert_array_equal(radii, st.radii)
    vis = st.radii > 0
    np.testing.assert_array_equal(state["cov3D"].view(np.uint32)[vis], st.cov3Ds.view(np.uint32)[vis])
    np.testing.assert_array_equal(state["clamped"][vis], st.clamped[vis])
    return S, g, st, grads


def _check(st, grads, label):
    dg = grads["_dgeom"]
    got = {k: v for k, v in grads.items() if k in pbc.GRAD_KEYS}
    np.testing.assert_array_equal(grads["means2D"][:, :2].view(np.uint32), np.asarray(dg[:, 0:2], np.float32).view(np.uint32))
    assert not grads["means2D"][:, 2].any()
    return pbc.assert_preprocess_per_element(st, got, dg, label=label)


@pytest.mark.parametrize("name", list(pbc.SCENES))
def test_scene_per_element(name):
    _, _, st, grads = _run(name)
    _check(st, grads, name)


@pytest.mark.parametrize("minb", [1, 4])
@pytest.mark.parametrize("staged", [0, 1, 2])
@pytest.mark.parametrize("name", ["P4099", "P31", "deg2", "aa_random", "sh3+x"])
def test_sh_staged_per_element(name, staged, minb):
    olds = {k: _lib.set_option(k, v) for k, v in (("sh_staged", staged), ("pre_bwd_minblocks", minb))}
    try:
        _, _, st, grads = _run(name)
    finally:
        for k, v in olds.items():
            _lib.set_option(k, v)
    _check(st, grads, f"{name} sh_staged {staged} minblocks {minb}")


def _factored_backward(S, g, dC, dD):
    """Forward through the rasterizer, then gms_rasterize_backward with RasterGrads.dL_dcolors_sh set (the factored SH
    gradient: no SH rows are written).  Returns the gradients and the kernel's record."""
    dev = "cuda"
    rasterizer.KEEP_DEBUG = True
    rs = gpu_settings(S, dev)
    t = {k: v.to(dev).float().contiguous() for k, v in g.items() if v is not None}
    P, M = t["means3D"].shape[0], t["shs"].shape[1]
    m2d = torch.zeros(P, 3, device=dev, requires_grad=True)       # a forward that a backward may follow
    _, radii, _ = dgr.GaussianRasterizer(raster_settings=rs)(means3D=t["means3D"], means2D=m2d, opacities=t["opacities"],
                                                              shs=t["shs"], scales=t["scales"], rotations=t["rotations"])
    dbg = rasterizer.last_debug
    keep = []
    s = rasterizer._settings_struct(rs, torch.device(dev), keep)
    i = rasterizer._inputs_struct(P, M, t["means3D"], t["opacities"], t["shs"], None, t["scales"], t["rotations"], None)
    saved = _lib.RasterSaved()
    b = dbg["scratch"].bufs
    p = rasterizer._ptr
    saved.geom, saved.binning, saved.image = p(b.get(_lib.BUF_GEOM)), p(b.get(_lib.BUF_BINNING)), p(b.get(_lib.BUF_IMAGE))
    saved.num_rendered = dbg["num_rendered"]
    saved.binning_capacity, saved.flags = dbg["bin_state"]
    e = lambda *shape: torch.full(shape, float("nan"), device=dev)
    out = dict(means3D=e(P, 3), means2D=e(P, 3), opacities=e(P, 1), scales=e(P, 3), rotations=e(P, 4), colors_sh=e(P, 3))
    gr = _lib.RasterGrads(p(out["means3D"]), p(out["means2D"]), p(out["opacities"]), None, None, p(out["scales"]),
                          p(out["rotations"]), None, p(out["colors_sh"]))
    gcol, gdep = torch.tensor(dC, device=dev), torch.tensor(dD, device=dev)[None]
    rc = _lib.lib().gms_rasterize_backward(C.byref(s), C.byref(i), radii.data_ptr(), C.byref(saved), gcol.data_ptr(),
                                           gdep.data_ptr(), C.byref(gr), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "gms_rasterize_backward")
    after = rasterizer.forward_debug_state(dbg["scratch"], dbg["num_rendered"], P, S.image_width, S.image_height, radii,
                                           bin_state=dbg["bin_state"])
    torch.cuda.synchronize()
    grads = {k: v.cpu().numpy() for k, v in out.items()}
    grads["_dgeom"] = after["dgeom"].cpu().numpy()
    return radii.cpu().numpy(), grads


@pytest.mark.parametrize("minb", [1, 4])
@pytest.mark.parametrize("name", ["P4099", "deg3", "aa_random", "sh2-y", "flat_edge_on"])
def test_factored_sh_gradient_per_element(name, minb):
    """The FACT arm of k_preprocess_bwd: the clamp-masked colour gradient against the reference's (bit for bit: budget 0),
    and the geometry gradients (whose SH view-direction term still reads the SH rows) within their budgets."""
    S, g = pbc.SCENES[name]()
    st = pbc.forward(S, g)
    old = _lib.set_option("pre_bwd_minblocks", minb)
    try:
        radii, grads = _factored_backward(S, g, *pbc.upstream(S))
    finally:
        _lib.set_option("pre_bwd_minblocks", old)
    np.testing.assert_array_equal(radii, st.radii)
    r = preprocess64.preprocess_backward64(st, grads["_dgeom"])
    assert not r["budget"]["dL_dcolors_sh"].any()
    _check(st, grads, f"{name} factored SH minblocks {minb}")
