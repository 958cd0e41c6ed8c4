"""Edge cases of the mesh -> Gaussian expansion (gms_expand_face_fwd / gms_expand_face_bwd) and their float64 reference.

One builder serves two runners: tests/test_hostshim_expansion_edges.py (the product's gms_expand.cuh compiled for the CPU)
and tests/test_gpu_expansion_edges.py (k_expand_fwd / k_expand_bwd).  Every case drives every output and every upstream
gradient at once; the reference is oracle/expansion.py run through autograd in float64, and the same oracle run in float32
measures how far plain fp32 arithmetic of the same formulas strays from it on each element.

Comparison rule (per element e of each output / gradient q):
    |kernel - f64| <= TOL[q] * max(err32, 2^-24 * (cond + floor_q))
err32 is how far the fp32 oracle strays from float64 on the element's face: the largest |oracle_fp32 - f64| over the
face's elements of q (an error of the face frame reaches every output of the face, and a single element's fp32 error can
be small by accident); for a vertex gradient, the sum of those errors over the faces around the vertex.
cond is the magnitude the element is formed from: |f64| itself; sum_j alpha_j |t_j| for xyz; the norm of the quaternion
row for a rotation component; (|dalpha_j| + sum_k |dalpha_k| alpha_k) / S for dL/d_alpha (the softmax-like normalisation
cancels); and for a vertex gradient the sum over the faces around the vertex of |that face's f64 contribution| (a vertex of
valence 2000 is a sum of 2000 atomics: its error scales with that sum, not with its value).  floor_q = 2^-10 * max|f64_q|
keeps elements that cancel to ~0 from demanding relative precision no fp32 evaluation has.

Branch-ambiguous faces.  The reference is discontinuous where rot_to_quat changes branch: which of the four quaternion
candidates is largest (`sel`) and the sign standardisation w >= 0.  A face is excluded from the per-element comparison when
  - the fp32 and float64 evaluations pick a different sel or a different sign, or
  - the two largest candidate magnitudes are within AMBIG_TIE (1e-5), or
  - the standardised |w| is below AMBIG_W (1e-5);
its Gaussians' rows, and every vertex it touches, then only have to be finite.  The runners print the count and bound it.

Zero-area faces (collinear, coincident corners) are a separate case: the eps = 1e-8 in |n| + eps, |a1| + eps, |u| + eps
makes their frame depend on rounding noise, so they are compared with the fp32 oracle, not with float64
(check_degenerate).
"""
from __future__ import annotations

import numpy as np
import torch

from gms_b200 import _lib, scenes
from oracle import expansion as oexp

EPS = 1e-8
AMBIG_TIE = 1e-5
AMBIG_W = 1e-5
AMBIG_MAX_FRACTION = 0.01
U24 = 2.0 ** -24

# bounds on the worst normalised error per quantity (see the comparison rule): 2-4x the worst measured over all cases on the
# CPU build and on an H100 (NVIDIA H100 80GB HBM3, 700 W power limit).  The large ones come from the sliver case
# (scaling_log 73, scaling_act 24, vertices 33: s2 = a2.v2 / 2 is a cancellation there) and from the K-fold sum of the
# scale gradient (19).
TOL = dict(alpha=4.0, xyz=8.0, scaling_log=150.0, rotation_raw=16.0, scaling_act=64.0, rotation_act=16.0, dL_dalpha_raw=12.0,
           dL_dscale_raw=48.0, dL_dvertices=96.0, dL_dtriangles=12.0)
TOL_DEGENERATE = 12.0

FACE_ROW_OUTPUTS = ("alpha", "xyz", "scaling_log", "rotation_raw", "scaling_act", "rotation_act", "dL_dalpha_raw", "dL_dscale_raw")


class Case:
    """vertices [V,3] float32, faces [F,3] int64, alpha_raw [F,K,3], scale_raw [F*K,1] and one upstream gradient per output.
    animated: the kernel reads triangles_in = vertices[faces] (every face has its own three vertices) and writes
    dL_dtriangles instead of scattering vertex gradients."""

    def __init__(self, name, vertices, faces, alpha_raw, scale_raw, seed, animated=False, degenerate=False,
                 max_ambiguous=AMBIG_MAX_FRACTION):
        self.name, self.animated, self.degenerate = name, animated, degenerate
        self.vertices = np.ascontiguousarray(vertices, np.float32)
        self.faces = np.ascontiguousarray(faces, np.int64)
        self.alpha_raw = np.ascontiguousarray(alpha_raw, np.float32)
        self.scale_raw = np.ascontiguousarray(scale_raw, np.float32).reshape(-1, 1)
        self.F, self.K = self.alpha_raw.shape[:2]
        self.P = self.F * self.K
        self.max_ambiguous = int(max_ambiguous * self.F)
        rs = np.random.RandomState(seed + 1000)
        self.up = {k: rs.randn(self.P, d).astype(np.float32) for k, d in
                   (("dL_dxyz", 3), ("dL_dscaling_log", 3), ("dL_drotation_raw", 4), ("dL_dscaling_act", 3), ("dL_drotation_act", 4))}
        assert self.faces.shape == (self.F, 3) and self.scale_raw.shape[0] == self.P

    def __repr__(self):
        return f"{self.name}(F={self.F}, K={self.K})"


# ---------------------------------------------------------------------------------------------------------- builders

def random_rotation(rs):
    q, r = np.linalg.qr(rs.randn(3, 3))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def trained_params(rs, F, K):
    """Parameters as Adam leaves them: alpha ~ N(0.3, 0.5) with whole rows <= 0 (they fall back to 1/3 each through the
    1e-8) and exact zeros (the ReLU kink); scale ~ N(0.8, 0.8) with negatives and exact zeros."""
    a = (0.3 + 0.5 * rs.randn(F, K, 3)).astype(np.float32)
    rows = rs.rand(F, K) < 0.05
    a[rows] = -np.abs(a[rows]) - 0.01
    a[rs.rand(F, K, 3) < 0.02] = 0.0
    s = (0.8 + 0.8 * rs.randn(F * K, 1)).astype(np.float32)
    s[rs.rand(F * K) < 0.03] = 0.0
    return a, s


def _sphere(level, rs, rotations=1, jitter=0.0, axis_scale=(1.0, 1.0, 1.0), scale=1.0):
    """`rotations` randomly rotated copies of icosphere(level), side by side, optionally jittered and scaled per axis."""
    v0, f0 = scenes.icosphere(level)
    vs, fs = [], []
    for r in range(rotations):
        v = v0.astype(np.float64) @ random_rotation(rs).T
        if jitter:
            v = v * (1.0 + jitter * rs.randn(*v.shape))
        v = v * np.asarray(axis_scale) @ random_rotation(rs).T
        vs.append(scale * (v + np.array([3.0 * r, 0.0, 0.0])))
        fs.append(f0 + r * v0.shape[0])
    return np.concatenate(vs).astype(np.float32), np.concatenate(fs)


def fan(n, rs):
    """n faces around one vertex: that vertex's gradient is a sum of n per-face terms.  The rim zigzags up and down so the
    faces are not slivers (an apex angle of 2 pi / n would make every face ill-conditioned)."""
    ang = (np.arange(n) + 0.3 * rs.rand(n)) * 2 * np.pi / n
    z = np.where(np.arange(n) % 2 == 0, 1.0, -1.0) * (0.8 + 0.4 * rs.rand(n))
    ring = np.stack([np.cos(ang), np.sin(ang), z], 1) * (1.0 + 0.1 * rs.rand(n, 1))
    v = np.concatenate([np.array([[0.0, 0.0, 0.1]]), ring]) @ random_rotation(rs).T
    f = np.stack([np.zeros(n, np.int64), 1 + np.arange(n), 1 + (np.arange(n) + 1) % n], 1)
    return v.astype(np.float32), f


def build_cases():
    rs = np.random.RandomState(2024)
    cases = []

    def add(name, v, f, K, animated=False, **kw):
        a, s = trained_params(rs, f.shape[0], K)
        if animated:
            v, f = v[f].reshape(-1, 3), np.arange(3 * f.shape[0]).reshape(-1, 3)
        cases.append(Case(name, v, f, a, s, seed=len(cases), animated=animated, **kw))

    add("rotations", *_sphere(2, rs, rotations=6), K=1)                   # 1920 faces: every quaternion branch and sign
    # axis-aligned: the faces on the icosahedron's mirror planes have two equal quaternion candidates or w = 0 exactly
    # (12 of 320: 10 ties, 2 with |w| ~ 1e-8)
    v, f = scenes.icosphere(2)
    add("unrotated", v.astype(np.float32), f, K=3, max_ambiguous=0.04)
    add("trained", *_sphere(2, rs, jitter=0.1), K=3)
    add("sliver", *_sphere(2, rs, axis_scale=(1.0, 1.0, 1e-3)), K=3)       # one axis squashed by 1e-3
    add("small", *_sphere(2, rs, jitter=0.05, scale=1e-3), K=7)
    add("large", *_sphere(2, rs, jitter=0.05, scale=1e3), K=7)
    add("jitter", *_sphere(1, rs, jitter=0.3), K=40)                       # K = 40: over the staging limit (direct kernel)
    add("fan", *fan(2003, rs), K=1)                                       # one vertex in 2003 faces
    add("animated", *_sphere(2, rs, rotations=2, jitter=0.1), K=3, animated=True)
    return cases


def degenerate_case():
    """Zero-area faces among regular ones: collinear corners (exact zero cross product in fp32), two coincident corners,
    all three coincident, and a corner at the centroid of the other two."""
    rs = np.random.RandomState(7)
    tris = [[[0, 0, 0], [1, 2, 3], [2, 4, 6]],            # collinear
            [[0.5, -1, 2], [0.5, -1, 2], [1, 0, 1]],     # t0 = t1
            [[1, 2, 3], [-1, 0, 2], [1, 2, 3]],          # t0 = t2
            [[0, 1, 0], [2, 1, 1], [2, 1, 1]],           # t1 = t2
            [[3, 3, 3], [3, 3, 3], [3, 3, 3]],           # all coincident
            [[-1, 0, 0], [1, 0, 0], [0, 0, 0]]]          # t2 at the midpoint of t0 t1
    reg = rs.randn(10, 3, 3)
    tri = np.concatenate([np.asarray(tris, np.float64), reg]).astype(np.float32)
    F, K = tri.shape[0], 3
    a, s = trained_params(rs, F, K)
    return Case("degenerate", tri.reshape(-1, 3), np.arange(3 * F).reshape(F, 3), a, s, seed=99, degenerate=True)


# ---------------------------------------------------------------------------------------------------------- reference

def _loss(out, up):
    xyz, sl, rr = out
    t = lambda k: torch.as_tensor(up[k]).to(xyz.dtype)
    return ((xyz * t("dL_dxyz")).sum() + (sl * t("dL_dscaling_log")).sum() + (rr * t("dL_drotation_raw")).sum() +
            (torch.exp(sl) * t("dL_dscaling_act")).sum() + (torch.nn.functional.normalize(rr) * t("dL_drotation_act")).sum())


def oracle_run(case, dtype):
    """oracle/expansion.py in `dtype` through autograd: every output, every gradient, and the per-face contributions to the
    corner gradients (dL/dtriangles)."""
    v = torch.tensor(case.vertices, dtype=dtype, requires_grad=True)
    a = torch.tensor(case.alpha_raw, dtype=dtype, requires_grad=True)
    s = torch.tensor(case.scale_raw, dtype=dtype, requires_grad=True)
    alpha, tri, xyz = oexp.update_alpha(a, v, torch.tensor(case.faces))
    tri.retain_grad()
    sl, rr = oexp.prepare_scaling_rot(tri, s, case.K, EPS)
    _loss((xyz, sl, rr), case.up).backward()
    d = lambda t: t.detach().numpy().astype(np.float64)
    out = dict(alpha=d(alpha), xyz=d(xyz), scaling_log=d(sl), rotation_raw=d(rr), scaling_act=d(torch.exp(sl)),
               rotation_act=d(torch.nn.functional.normalize(rr)), dL_dalpha_raw=d(a.grad), dL_dscale_raw=d(s.grad),
               dL_dtriangles=d(tri.grad).reshape(-1, 9), dL_dvertices=d(v.grad))
    out["_rows"] = oexp.face_frames(tri.detach(), EPS)[0]
    # magnitudes the elements are formed from (see `cond` in the module docstring)
    t = tri.detach()
    out["_cond_xyz"] = d(torch.matmul(alpha.detach(), t.abs()).reshape(-1, 3))
    dal = torch.einsum("fkc,fjc->fkj", torch.as_tensor(case.up["dL_dxyz"]).to(dtype).reshape(case.F, case.K, 3), t).abs()
    r = torch.relu(a.detach()) + 1e-8
    S = r.sum(-1, keepdim=True)
    out["_cond_alpha"] = d((dal + (dal * r / S).sum(-1, keepdim=True)) / S)
    return out


def quat_branch(rows):
    """(sel, sign of the un-standardised w, gap between the two largest candidate magnitudes, standardised |w|) per face,
    in the dtype of `rows` (face_frames' rows; the rotation's columns)."""
    m = rows.transpose(-2, -1)
    d0, d1, d2 = m[:, 0, 0], m[:, 1, 1], m[:, 2, 2]
    arg = torch.stack((1 + d0 + d1 + d2, 1 + d0 - d1 - d2, 1 - d0 + d1 - d2, 1 - d0 - d1 + d2), -1)
    mag = torch.sqrt(arg.clamp(min=0))
    sel = mag.argmax(-1)
    top = mag.sort(-1, descending=True).values
    w_num = torch.stack((mag[:, 0] ** 2, m[:, 2, 1] - m[:, 1, 2], m[:, 0, 2] - m[:, 2, 0], m[:, 1, 0] - m[:, 0, 1]), -1)
    w = w_num[torch.arange(m.shape[0]), sel] / (2 * mag.max(-1).values.clamp(min=0.1))
    return sel.numpy(), (w < 0).numpy(), (top[:, 0] - top[:, 1]).numpy(), w.abs().numpy()


class Reference:
    def __init__(self, case):
        self.case = case
        self.f64 = oracle_run(case, torch.float64)
        self.f32 = oracle_run(case, torch.float32)
        s64, n64, gap, w = quat_branch(self.f64["_rows"])
        s32, n32, _, _ = quat_branch(self.f32["_rows"])
        self.sel64, self.neg64 = s64, n64
        self.amb_face = (s64 != s32) | (n64 != n32) | (gap < AMBIG_TIE) | (w < AMBIG_W)
        if case.degenerate:
            self.amb_face[:] = False
        amb_v = np.zeros(case.vertices.shape[0], bool)
        amb_v[case.faces[self.amb_face].reshape(-1)] = True
        self.amb_vertex = amb_v
        # cond of a vertex gradient: sum over its faces of |that face's contribution|
        cv = np.zeros_like(self.f64["dL_dvertices"])
        np.add.at(cv, case.faces.reshape(-1), np.abs(self.f64["dL_dtriangles"]).reshape(-1, 3))
        qn = lambda q: np.broadcast_to(np.linalg.norm(q, axis=1, keepdims=True), q.shape)
        self.cond = dict(xyz=self.f64["_cond_xyz"], dL_dalpha_raw=self.f64["_cond_alpha"], dL_dvertices=cv,
                         rotation_raw=qn(self.f64["rotation_raw"]), rotation_act=qn(self.f64["rotation_act"]))

    def fp32_error(self, q, shape):
        """How far fp32 arithmetic of the same formulas strays from float64 on each element of q: the largest
        |oracle_fp32 - f64| over the element's face (an error of the face frame reaches every output of the face, and one
        element's fp32 error can be small by accident); for a vertex gradient, the sum of those of its faces' corners."""
        err = np.abs(self.f32[q] - self.f64[q]).reshape(shape)
        if q == "dL_dvertices":
            acc = np.zeros_like(err)
            np.add.at(acc, self.case.faces.reshape(-1), np.abs(self.f32["dL_dtriangles"] - self.f64["dL_dtriangles"]).reshape(-1, 3))
            return np.maximum(err, acc)
        per_face = err.reshape(self.case.F, -1)
        return np.broadcast_to(per_face.max(axis=1, keepdims=True), per_face.shape).reshape(shape)

    @property
    def n_ambiguous(self):
        return int(self.amb_face.sum())

    def row_mask(self, q):
        """rows of output q that must match per element (False: a branch-ambiguous face's rows / vertices)."""
        if q == "dL_dvertices":
            return ~self.amb_vertex
        if q == "dL_dtriangles":
            return ~self.amb_face
        return np.repeat(~self.amb_face, self.case.K)


# ---------------------------------------------------------------------------------------------------------- kernel runner

OUT_SHAPES = dict(alpha=3, triangles=9, xyz=3, scaling_log=3, rotation_raw=4, scaling_act=3, rotation_act=4)


def run_abi(case, put, get, forward, backward):
    """Both expansion entry points on `case` through the C ABI structs, every output and upstream gradient at once.
    put(np.ndarray) -> (buffer, address) places an array where the kernels read it; get(buffer) -> np.ndarray reads it
    back; forward(args) / backward(args, grads) make the calls.  Returns {output name: float64 array, rows first}."""
    keep = []

    def place(arr):
        buf, addr = put(np.ascontiguousarray(arr))
        keep.append(buf)
        return buf, addr

    F, K, P = case.F, case.K, case.P
    a = _lib.ExpandArgs()
    a.V, a.F, a.K, a.eps = case.vertices.shape[0], F, K, EPS
    if case.animated:
        a.V = 0
        _, a.triangles_in = place(case.vertices[case.faces].reshape(F, 9))
    else:
        _, a.vertices = place(case.vertices)
        _, a.faces = place(case.faces)
    _, a.alpha_raw = place(case.alpha_raw)
    _, a.scale_raw = place(case.scale_raw)
    outs = {}
    for k, w in OUT_SHAPES.items():
        rows = F if k == "triangles" else P
        outs[k], addr = place(np.full((rows, w), np.nan, np.float32))
        setattr(a, k, addr)
    forward(a)
    res = {k: get(b).astype(np.float64) for k, b in outs.items()}
    res["alpha"] = res["alpha"].reshape(F, K, 3)
    # backward: the output pointers are not read
    for k in OUT_SHAPES:
        setattr(a, k, None)
    g = _lib.ExpandGrads()
    for k, arr in case.up.items():
        _, addr = place(arr)
        setattr(g, k, addr)
    grads = dict(dL_dalpha_raw=np.full((F, K, 3), np.nan, np.float32), dL_dscale_raw=np.full((P, 1), np.nan, np.float32))
    if case.animated:
        grads["dL_dtriangles"] = np.full((F, 9), np.nan, np.float32)
    else:
        grads["dL_dvertices"] = np.zeros_like(case.vertices)
    bufs = {}
    for k, arr in grads.items():
        bufs[k], addr = place(arr)
        setattr(g, k, addr)
    backward(a, g)
    res.update({k: get(b).astype(np.float64) for k, b in bufs.items()})
    return res


# ---------------------------------------------------------------------------------------------------------- comparison

def check_case(ref, got, tol, label):
    """Per-element comparison (module docstring).  Returns {quantity: worst normalised error} and prints it."""
    case = ref.case
    np.testing.assert_array_equal(got["triangles"].reshape(-1, 3, 3), case.vertices[case.faces])
    qs = [q for q in FACE_ROW_OUTPUTS] + ["dL_dtriangles" if case.animated else "dL_dvertices"]
    worst = {}
    for q in qs:
        g = got[q].reshape(-1, 9 if q == "dL_dtriangles" else got[q].shape[-1])
        r64 = ref.f64[q].reshape(g.shape)
        assert np.isfinite(g).all(), f"{label} {q}: non-finite values"
        ok = ref.row_mask(q)
        cond = np.abs(ref.cond.get(q, r64)).reshape(g.shape)
        floor = 2.0 ** -10 * float(np.abs(r64).max())
        bound = np.maximum(ref.fp32_error(q, g.shape), U24 * (cond + floor))
        e = (np.abs(g - r64) / bound)[ok]
        worst[q] = float(e.max()) if e.size else 0.0
    n_amb = ref.n_ambiguous
    print(f"[expand-edges] {label}: ambiguous faces {n_amb}/{case.F}; worst |kernel-f64| / max(|fp32-f64|, 2^-24 (cond+floor)): " +
          ", ".join(f"{q} {v:.2f}" for q, v in worst.items()))
    assert n_amb <= case.max_ambiguous, f"{label}: {n_amb} branch-ambiguous faces of {case.F}"
    for q, v in worst.items():
        assert v <= tol[q], f"{label} {q}: normalised error {v:.3g} > {tol[q]}"
    return worst


def check_degenerate(ref, got, tol, label, frame_outputs=True):
    """Zero-area faces: every output and gradient finite, and equal to the fp32 oracle within tol * 2^-24 * max|fp32| per
    quantity.  frame_outputs=False compares only what does not depend on the in-plane axes of the frame (alpha, xyz, their
    gradient, scaling columns 0 and 1): of a zero-area face, |u| + eps is a few eps, so the rotation, scaling column 2 and
    the vertex / scale gradients through them are decided by rounding, and FMA contraction (GPU) rounds differently from
    the oracle."""
    worst = {}
    for q in FACE_ROW_OUTPUTS + ("dL_dvertices",):
        g = got[q].reshape(-1, got[q].shape[-1])
        r32 = ref.f32[q].reshape(g.shape)
        assert np.isfinite(g).all() and np.isfinite(r32).all(), f"{label} {q}: non-finite values"
        if not frame_outputs:
            if q in ("scaling_log", "scaling_act"):
                g, r32 = g[:, :2], r32[:, :2]
            elif q not in ("alpha", "xyz", "dL_dalpha_raw"):
                continue
        scale = max(float(np.abs(r32).max()), 1e-30)
        worst[q] = float(np.abs(g - r32).max() / (U24 * scale))
    print(f"[expand-edges] {label}: worst |kernel-fp32 oracle| / (2^-24 max|fp32 oracle|): " +
          ", ".join(f"{q} {v:.1f}" for q, v in worst.items()))
    for q, v in worst.items():
        assert v <= tol, f"{label} {q}: {v:.3g} > {tol}"
    return worst


def branch_coverage(refs):
    """Every quaternion branch sel = 0..3 and both standardisation signs occur on some unambiguous face (float64)."""
    sel = np.concatenate([r.sel64[~r.amb_face] for r in refs])
    neg = np.concatenate([r.neg64[~r.amb_face] for r in refs])
    counts = np.bincount(sel, minlength=4)
    print(f"[expand-edges] quaternion branches over all cases: sel counts {counts.tolist()}, negative w before "
          f"standardisation {int(neg.sum())} of {neg.size}")
    assert (counts > 0).all() and neg.any() and (~neg).any()
    # every branch with both signs (sel = 0 has w = |q|^2 / D > 0 by construction)
    for s in (1, 2, 3):
        assert neg[sel == s].any() and (~neg[sel == s]).any(), f"branch {s} misses a sign"
