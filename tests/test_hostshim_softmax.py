"""The product's softmax expansion (csrc/gms_expand.cuh, compiled for the CPU by tests/hostshim, selected through
gms_expand_args.alpha_activation) against float64: the weights and their backward on rows with logits up to +/-1e3, exact
ties and one dominant weight; and the face frame, scales and rotations bit for bit those of the relu weights."""
import ctypes as C

import numpy as np
import pytest

from gms_b200 import _lib
from hostshim import build_shim

U = 2.0 ** -24


@pytest.fixture(scope="module")
def shim():
    return C.CDLL(build_shim.build())


def _mesh(rs, F):
    v = rs.randn(F * 3, 3).astype(np.float32)
    return v, np.arange(3 * F, dtype=np.int64).reshape(F, 3)


def _logits(rs, F, K):
    a = (rs.randn(F, K, 3) * 4).astype(np.float32)
    a[0] = np.float32(1e3) * np.sign(rs.randn(K, 3)).astype(np.float32)        # +/- 1e3
    a[1] = np.float32(2.5)                                                     # exact three-way ties
    a[2, :, 0], a[2, :, 1], a[2, :, 2] = 1e3, -1e3, 0.0                        # one dominant weight
    a[3] = np.float32(1e3) + rs.rand(K, 3).astype(np.float32)                  # far above expf's range without the max
    a[4, :, :2] = np.float32(-1e3)                                             # two equal minima
    return a


def _run(shim, v, f, a, s, up, act):
    F, K = a.shape[:2]
    P = F * K
    keep = []
    ptr = lambda arr: (keep.append(arr), arr.ctypes.data)[1]
    args = _lib.ExpandArgs()
    args.V, args.F, args.K, args.eps, args.alpha_activation = v.shape[0], F, K, 1e-8, act
    args.vertices, args.faces, args.alpha_raw, args.scale_raw = ptr(v), ptr(f), ptr(a), ptr(s)
    out = {k: np.full((P, w), np.nan, np.float32) for k, w in (("alpha", 3), ("xyz", 3), ("scaling_act", 3), ("rotation_act", 4))}
    for k, arr in out.items():
        setattr(args, k, ptr(arr))
    assert shim.shim_expand_forward(C.byref(args)) == 0
    for k in out:
        setattr(args, k, None)
    g = _lib.ExpandGrads()
    g.dL_dxyz, g.dL_dscaling_act, g.dL_drotation_act = ptr(up[0]), ptr(up[1]), ptr(up[2])
    grads = dict(dL_dalpha_raw=np.full((P, 3), np.nan, np.float32), dL_dscale_raw=np.full((P, 1), np.nan, np.float32),
                 dL_dvertices=np.zeros_like(v))
    for k, arr in grads.items():
        setattr(g, k, ptr(arr))
    assert shim.shim_expand_backward(C.byref(args), C.byref(g)) == 0
    out.update(grads)
    return out


def test_softmax_weights_and_backward_vs_float64(shim):
    rs = np.random.RandomState(5)
    F, K = 40, 7
    v, f = _mesh(rs, F)
    a = _logits(rs, F, K)
    s = np.abs(rs.randn(F * K, 1)).astype(np.float32)
    up = (rs.randn(F * K, 3).astype(np.float32), rs.randn(F * K, 3).astype(np.float32), rs.randn(F * K, 4).astype(np.float32))
    got = _run(shim, v, f, a, s, up, _lib.ALPHA_SOFTMAX)
    x = a.astype(np.float64).reshape(-1, 3)
    e = np.exp(x - x.max(1, keepdims=True))
    al = e / e.sum(1, keepdims=True)
    assert np.isfinite(got["alpha"]).all() and np.isfinite(got["dL_dalpha_raw"]).all()
    # x_j - m is rounded once: exp carries that relative error times |x_j - m| into e_j, and through s into every weight
    d = np.abs(x - x.max(1, keepdims=True))
    c = 8 + d + (al * d).sum(1, keepdims=True)
    err = np.abs(got["alpha"] - al)
    worst = float((err / (U * al * c + 1e-45)).max())
    print(f"[softmax-shim] worst |alpha - f64| / (2^-24 alpha (8 + |x - m| + sum alpha |x - m|)): {worst:.3f}")
    assert worst <= 2.0
    # exact ties give exactly 1/3 each; a dominant logit gives exactly (1, 0, 0)
    np.testing.assert_array_equal(got["alpha"].reshape(F, K, 3)[1], np.float32(1) / np.float32(3))
    np.testing.assert_array_equal(got["alpha"].reshape(F, K, 3)[2], np.broadcast_to(np.float32([1, 0, 0]), (K, 3)))
    # xyz = alpha @ triangle
    t = v[f].astype(np.float64)                                                  # [F,3,3]
    xyz = np.einsum("fkj,fjc->fkc", al.reshape(F, K, 3), t).reshape(-1, 3)
    cond = np.einsum("fkj,fjc->fkc", al.reshape(F, K, 3), np.abs(t)).reshape(-1, 3)
    assert (np.abs(got["xyz"] - xyz) <= 8 * U * cond + 1e-30).all()
    # dL/d_alpha_j = alpha_j (g_j - sum_i alpha_i g_i), g_j = dL/dxyz . t_j; bound scaled by alpha_j (G_j + sum_i alpha_i G_i)
    dx = up[0].astype(np.float64).reshape(F, K, 3)
    g = np.einsum("fkc,fjc->fkj", dx, t).reshape(-1, 3)
    G = np.einsum("fkc,fjc->fkj", np.abs(dx), np.abs(t)).reshape(-1, 3)
    ref = al * (g - (al * g).sum(1, keepdims=True))
    bound = 16 * U * al * (G + (al * G).sum(1, keepdims=True)) + 2 * U * al * (c * np.abs(g - (al * g).sum(1, keepdims=True)) +
                                                                           (al * c * np.abs(g)).sum(1, keepdims=True)) + 1e-38
    worst = float((np.abs(got["dL_dalpha_raw"] - ref) / bound).max())
    print(f"[softmax-shim] worst |dL/d_alpha - f64| / bound: {worst:.3f}")
    assert worst <= 1.0
    # the frame does not see the activation: scales and rotations are the relu run's, bit for bit, and so is dL/d_scale
    rel = _run(shim, v, f, a, s, up, _lib.ALPHA_RELU)
    for k in ("scaling_act", "rotation_act", "dL_dscale_raw"):
        np.testing.assert_array_equal(got[k], rel[k], err_msg=k)
