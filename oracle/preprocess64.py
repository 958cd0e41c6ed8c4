"""The preprocess backward (stage 2 of the rasterizer's backward) in float64, with an a-priori error budget per element.

TEST INFRASTRUCTURE ONLY.  `preprocess_backward64(st, dgeom)` restates the operation that gms_preprocess_backward_geom and
gms_sh_backward (csrc/gms_preprocess.cuh) and gmso_preprocess_backward (gms_oracle.c) implement: the upstream
diff-gaussian-rasterization backward, not the true derivative of the forward.  The two differ where the upstream does:
  * dL/dtz treats the guard-band-clamped tx, ty as constants (the 2 fx tx / tz^3 term),
  * 1e-7 is added to det^2 in the conic gradient (the forward has no such term),
and the conic xy gradient is in the upstream's half convention.  The SH constants, the 0.3 px dilation and every other
constant are their fp32 values: they are part of the operation.

Soundness of the budget (running-error analysis, applied mechanically).  Every intermediate is a pair
(v, b): v its value in float64, b a bound on |x - v| for ANY fp32 evaluation x of the same expression tree on the same fp32
inputs, with each operation rounded to nearest (or fused with its neighbour).  Inputs are exact (b = 0; 2^-126 for a
subnormal input, which a flush-to-zero build reads as 0).  For each operation on (x, bx), (y, by):
  x +- y:  bx + by                                   (exact)
  x * y:   |x| by + |y| bx + bx by                   (exact)
  x / y:   (bx + |x / y| by) / max(|y| - by, L)      (exact; L a known lower bound of |y|, else 0 -> infinite)
  sqrt x:  min(bx / sqrt x, sqrt bx)                 (exact, x >= 0)
  sqrt max(x, c):  max(sqrt v' - sqrt max(c, v - b), sqrt max(c, v + b) - sqrt v'),  v' = max(v, c)
                                                     (exact, c > 0; every evaluation is >= fl(sqrt c) >= sqrt(c) (1 - U))
  -x, select:  b unchanged                           (no rounding)
and then the rounding of the result is added: U (|v| + b) + [|v| + b > 0] 2^-126.  The first term bounds the rounding to
nearest of a value within b of v; the second the absolute error of a subnormal result or of its flush to zero.  An FMA
drops the rounding of its product, so the bound of the unfused tree also covers any contraction (nvcc contracts, the C
oracle and the host shim are built with -ffp-contract=off).  U = 2^-24 (1 + 2^-20): the 2^-20 covers the float64 rounding of
v itself, which is 2^-29 of the fp32 rounding at every step.  The expression tree is the product's (gms_preprocess.cuh); an
implementation that associates a product chain differently gets the same relative bound, and the C oracle's other
summation order of the SH view-direction term is checked against this budget by the tests.  An operation whose exact
result is 0 from exact inputs adds nothing, so a Gaussian with a zero record has budget 0 and must come out exactly 0.
fp32 overflow is not modelled: outside the det^2 select below it would make the implementation's output infinite or NaN,
which the tests reject on their own.

Branches.  Three decisions are the fp32 forward's: the guard-band clamp (|tx/tz| > 1.3 tan fov, per axis), the
antialiasing test ratio > 2.5e-5, and the det^2 overflow select (det^2 + 1e-7 <= FLT_MAX).  Each is decided here on the
float64 value; a Gaussian whose value lies within its bound of the threshold is AMBIGUOUS: an fp32 evaluation may take the
other branch.  The reference is then also evaluated with that one decision flipped, and its budget becomes the larger
of the two bounds plus |branch A - branch B|, element by element (as the composite budget does for flip candidates).
The SH colour clamp is not decided here: the forward's mask (st.clamped) is an input of the backward.
"""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24 * (1.0 + 2.0 ** -20)
TINY = 2.0 ** -126
F32_MAX = float(np.finfo(np.float32).max)


def f32(c):
    return float(np.float32(c))


HVAR = f32(0.3)
AA_FLOOR = f32(0.000025)
EPS_W = f32(0.0000001)        # phom.w + 1e-7 (forward and backward) and det^2 + 1e-7 (backward only)
SH_C0 = f32(0.28209479177387814)
SH_C1 = f32(0.4886025119029199)
SH_C2 = [f32(c) for c in (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792,
                          0.5462742152960396)]
SH_C3 = [f32(c) for c in (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
                          -0.4570457994644658, 1.445305721320277, -0.5900435899266435)]


class E:
    """A float64 value and a bound on |any fp32 evaluation - value| (see the module docstring), elementwise over arrays."""
    __array_ufunc__ = None       # numpy operands defer to E's reflected operators
    __slots__ = ("v", "b", "lo")

    def __init__(self, v, b=None, lo=0.0):
        self.v = np.asarray(v, np.float64)
        self.b = np.zeros_like(self.v) if b is None else np.asarray(b, np.float64)
        self.lo = lo        # a lower bound of |any evaluation| when one is known (a floored square root), else 0

    @staticmethod
    def input(a):
        a = np.asarray(a, np.float64)
        return E(a, np.where((a != 0) & (np.abs(a) < TINY), TINY, 0.0))

    @staticmethod
    def _r(v, b):
        m = np.abs(v) + b
        return E(v, b + U * m + np.where(m > 0, TINY, 0.0))

    def __add__(self, o):
        o = lift(o)
        return E._r(self.v + o.v, self.b + o.b)

    def __sub__(self, o):
        o = lift(o)
        return E._r(self.v - o.v, self.b + o.b)

    def __mul__(self, o):
        if isinstance(o, float):        # an exact constant keeps a known lower bound, less one rounding
            r = E._r(self.v * o, np.abs(o) * self.b)
            r.lo = self.lo * abs(o) * (1.0 - U)
            return r
        o = lift(o)
        return E._r(self.v * o.v, np.abs(self.v) * o.b + np.abs(o.v) * self.b + self.b * o.b)

    def __truediv__(self, o):
        o = lift(o)
        with np.errstate(divide="ignore", invalid="ignore"):
            q = self.v / o.v
            den = np.maximum(np.abs(o.v) - o.b, o.lo)
            b = np.where(den > 0, (self.b + np.abs(q) * o.b) / np.where(den > 0, den, 1.0), np.inf)
        return E._r(q, b)

    __radd__ = __add__
    __rmul__ = __mul__

    def __rsub__(self, o):
        return lift(o) - self

    def __rtruediv__(self, o):
        return lift(o) / self

    def __neg__(self):
        return E(-self.v, self.b)


def lift(x):
    return x if isinstance(x, E) else E(x)


class _E64:
    """Backend of the budgeted float64 evaluation."""
    inp = staticmethod(E.input)
    const = staticmethod(lambda c: E(c))

    @staticmethod
    def sqrt(x):
        v = np.sqrt(np.maximum(x.v, 0.0))
        with np.errstate(divide="ignore", invalid="ignore"):
            b = np.minimum(np.where(v > 0, x.b / np.where(v > 0, v, 1.0), np.inf), np.sqrt(x.b))
        return E._r(v, b)

    @staticmethod
    def sqrt_floor(x, c):
        """sqrt(max(x, c)), c > 0: every evaluation lies in [sqrt(max(c, v - b)), sqrt(v + b)], which keeps the bound of a
        square root near the floor below its value (a later division by it stays finite)."""
        v = np.sqrt(np.maximum(x.v, c))
        lo, hi = np.sqrt(np.maximum(c, x.v - x.b)), np.sqrt(np.maximum(c, x.v + x.b))
        r = E._r(v, np.maximum(v - lo, hi - v))
        r.lo = np.sqrt(c) * (1.0 - U)
        return r

    @staticmethod
    def where(m, x, y):
        x, y = lift(x), lift(y)
        return E(np.where(m, x.v, y.v), np.where(m, x.b, y.b))

    val = staticmethod(lambda x: x.v)
    bnd = staticmethod(lambda x: x.b)


class _F32:
    """Backend of a plain fp32 evaluation of the same expression tree (numpy rounds every float32 operation)."""
    inp = staticmethod(lambda a: np.asarray(a, np.float32))
    const = staticmethod(np.float32)
    sqrt = staticmethod(lambda x: np.sqrt(x).astype(np.float32))
    sqrt_floor = staticmethod(lambda x, c: np.sqrt(np.maximum(x, np.float32(c))).astype(np.float32))
    where = staticmethod(lambda m, x, y: np.where(m, x, y).astype(np.float32))
    val = staticmethod(lambda x: np.asarray(x, np.float64))
    bnd = staticmethod(lambda x: np.zeros(np.shape(x)))


BUGS = ("no_xmul", "conic_full", "no_aa_ratio", "no_sh_dir", "view_transposed", "drot_sign")


def _dot3(a0, b0, a1, b1, a2, b2):
    return (a0 * b0 + a1 * b1) + a2 * b2


def _evaluate(X, I, force=None, bug=None, det2_eps=EPS_W):
    """One evaluation of the backward for every Gaussian of I (visible ones only) under backend X.  `force` maps a decision
    name to the boolean array to use instead of the backend's own decision.  Returns (outputs, decision quantities)."""
    force = force or {}
    P = I["P"]
    inp = X.inp
    view, proj = [float(v) for v in I["view"]], [float(v) for v in I["proj"]]
    mean = [inp(I["means"][:, k]) for k in range(3)]
    cov6 = [inp(I["cov6"][:, k]) for k in range(6)]
    g = I["dgeom"]
    g2x, g2y, dcx, dcy, dcz, dop = (inp(g[:, k]) for k in range(6))
    dcol = [inp(g[:, 6 + k]) for k in range(3)]
    dinv = inp(g[:, 9])
    fx, fy = I["focal_x"], I["focal_y"]
    dec = {}

    def decide(name, q, thr, above):
        """above(value) -> branch; ambiguous where |value - thr| <= bound."""
        v, b = X.val(q), X.bnd(q)
        dec[name] = (above(v), np.abs(np.abs(v) - thr) <= b if name in ("xclamp", "yclamp") else np.abs(v - thr) <= b)
        return force.get(name, dec[name][0])

    # view-space point and the EWA Jacobian (gms_cov2d)
    pv = [_dot3(view[r], mean[0], view[4 + r], mean[1], view[8 + r], mean[2]) + view[12 + r] for r in range(3)]
    tz = pv[2]
    limx, limy = f32(np.float32(1.3) * np.float32(I["tanfovx"])), f32(np.float32(1.3) * np.float32(I["tanfovy"]))
    txtz, tytz = pv[0] / tz, pv[1] / tz
    clx = decide("xclamp", txtz, limx, lambda v: np.abs(v) > limx)
    cly = decide("yclamp", tytz, limy, lambda v: np.abs(v) > limy)
    sx, sy = np.where(X.val(txtz) < 0, -limx, limx), np.where(X.val(tytz) < 0, -limy, limy)
    tx = X.where(clx, X.inp(sx), txtz) * tz
    ty = X.where(cly, X.inp(sy), tytz) * tz
    xmul, ymul = X.inp(np.where(clx, 0.0, 1.0)), X.inp(np.where(cly, 0.0, 1.0))
    if bug == "no_xmul":
        xmul = ymul = X.inp(np.ones(P))
    tz2 = tz * tz
    J00, J02 = fx / tz, -(fx * tx) / tz2
    J11, J12 = fy / tz, -(fy * ty) / tz2
    M0 = [J00 * view[4 * j] + J02 * view[4 * j + 2] for j in range(3)]
    M1 = [J11 * view[4 * j + 1] + J12 * view[4 * j + 2] for j in range(3)]
    S00, S01, S02, S11, S12, S22 = cov6
    v0 = _dot3(S00, M0[0], S01, M0[1], S02, M0[2]); v1 = _dot3(S01, M0[0], S11, M0[1], S12, M0[2])
    v2 = _dot3(S02, M0[0], S12, M0[1], S22, M0[2])
    w0 = _dot3(S00, M1[0], S01, M1[1], S02, M1[2]); w1 = _dot3(S01, M1[0], S11, M1[1], S12, M1[2])
    w2 = _dot3(S02, M1[0], S12, M1[1], S22, M1[2])
    a0 = _dot3(M0[0], v0, M0[1], v1, M0[2], v2)
    b = _dot3(M1[0], v0, M1[1], v1, M1[2], v2)
    c0 = _dot3(M1[0], w0, M1[1], w1, M1[2], w2)

    # gms_preprocess_backward_geom
    a, c = a0 + HVAR, c0 + HVAR
    det_cov = a0 * c0 - b * b
    det = a * c - b * b
    zero = X.inp(np.zeros(P))
    dL_da = dL_db = dL_dc = zero
    if I["antialiasing"]:
        ratio = det_cov / det
        h = X.sqrt_floor(ratio, AA_FLOOR)
        dopacity = dop * h
        aa = decide("aa", ratio, AA_FLOOR, lambda v: v > AA_FLOOR)
        if bug != "no_aa_ratio":
            dL_dratio = (dop * I["opac"]) / (2.0 * h)
            inv_det = 1.0 / det
            k = dL_dratio * inv_det * inv_det
            dL_da = X.where(aa, k * (c0 * det - det_cov * c), zero)
            dL_dc = X.where(aa, k * (a0 * det - det_cov * a), zero)
            dL_db = X.where(aa, k * ((-2.0 * b) * det + (2.0 * b) * det_cov), zero)
    else:
        dopacity = dop
    denom = det
    with np.errstate(over="ignore"):
        denom2 = denom * denom + det2_eps
    ovf = decide("ovf", denom2, F32_MAX, lambda v: v > F32_MAX)
    if bug == "conic_full":
        dcy = 0.5 * dcy
    with np.errstate(over="ignore", invalid="ignore"):
        d2i = 1.0 / X.where(ovf, X.inp(np.ones(P)), denom2)
        ta = d2i * (((-c) * c * dcx + (2.0 * b) * c * dcy) + (denom - a * c) * dcz)
        tc = d2i * (((-a) * a * dcz + (2.0 * a) * b * dcy) + (denom - a * c) * dcx)
        tb = (d2i * 2.0) * ((b * c * dcx - (denom + (2.0 * b) * b) * dcy) + a * b * dcz)
    dL_da = dL_da + X.where(ovf, zero, ta)
    dL_dc = dL_dc + X.where(ovf, zero, tc)
    dL_db = dL_db + X.where(ovf, zero, tb)

    g6 = [None] * 6
    for k, j in ((0, 0), (3, 1), (5, 2)):
        g6[k] = (M0[j] * M0[j] * dL_da + M0[j] * M1[j] * dL_db) + M1[j] * M1[j] * dL_dc
    for k, (i, j) in ((1, (0, 1)), (2, (0, 2)), (4, (2, 1))):
        g6[k] = ((2.0 * M0[i]) * M0[j] * dL_da + (M0[min(i, j)] * M1[max(i, j)] + M0[max(i, j)] * M1[min(i, j)]) * dL_db) + \
            (2.0 * M1[min(i, j)]) * M1[max(i, j)] * dL_dc
    S = [cov6[0], cov6[1], cov6[2], cov6[1], cov6[3], cov6[4], cov6[2], cov6[4], cov6[5]]
    u0 = [(2.0 * dL_da) * M0[j] + dL_db * M1[j] for j in range(3)]
    u1 = [(2.0 * dL_dc) * M1[j] + dL_db * M0[j] for j in range(3)]
    dM0 = [(u0[0] * S[j] + u0[1] * S[3 + j]) + u0[2] * S[6 + j] for j in range(3)]
    dM1 = [(u1[0] * S[j] + u1[1] * S[3 + j]) + u1[2] * S[6 + j] for j in range(3)]
    dJ00 = (dM0[0] * view[0] + dM0[1] * view[4]) + dM0[2] * view[8]
    dJ02 = (dM0[0] * view[2] + dM0[1] * view[6]) + dM0[2] * view[10]
    dJ11 = (dM1[0] * view[1] + dM1[1] * view[5]) + dM1[2] * view[9]
    dJ12 = (dM1[0] * view[2] + dM1[1] * view[6]) + dM1[2] * view[10]
    tzi = 1.0 / tz
    tzi2 = tzi * tzi
    tzi3 = tzi2 * tzi
    dL_dtx = (xmul * -fx) * tzi2 * dJ02
    dL_dty = (ymul * -fy) * tzi2 * dJ12
    dL_dtz = ((-fx * tzi2 * dJ00 - fy * tzi2 * dJ11) + (2.0 * fx * tx) * tzi3 * dJ02) + (2.0 * fy * ty) * tzi3 * dJ12
    dL_dtz = dL_dtz - dinv / (tz * tz)
    # transformVec4x3Transpose: dmean = W^T dt (view[4 * c + r] = W[r][c])
    Wt = (lambda r, c: view[4 * c + r]) if bug == "view_transposed" else (lambda r, c: view[4 * r + c])
    dm = [(Wt(i, 0) * dL_dtx + Wt(i, 1) * dL_dty) + Wt(i, 2) * dL_dtz for i in range(3)]
    ph = [_dot3(proj[r], mean[0], proj[4 + r], mean[1], proj[8 + r], mean[2]) + proj[12 + r] for r in range(4)]
    m_w = 1.0 / (ph[3] + EPS_W)
    mul1, mul2 = ph[0] * m_w * m_w, ph[1] * m_w * m_w
    for i in range(3):
        dm[i] = dm[i] + ((proj[4 * i] * m_w - proj[4 * i + 3] * mul1) * g2x + (proj[4 * i + 1] * m_w - proj[4 * i + 3] * mul2) * g2y)

    out = dict(dL_dcov3D=g6, dL_dopacity=[dopacity])
    gmask = [X.where(I["clamped"][:, ch] != 0, zero, dcol[ch]) for ch in range(3)]
    if I["shs"] is not None:
        D, M = I["D"], I["M"]
        nc = (D + 1) ** 2
        sh = I["shs"]
        cp = [float(v) for v in I["campos"]]
        vv = [mean[k] - cp[k] for k in range(3)]
        ln = X.sqrt((vv[0] * vv[0] + vv[1] * vv[1]) + vv[2] * vv[2])
        x, y, z = (vv[k] / ln for k in range(3))
        C1, C2, C3 = X.const(SH_C1), [X.const(cc) for cc in SH_C2], [X.const(cc) for cc in SH_C3]
        B = [X.inp(np.full(P, SH_C0))] + [None] * 15
        t = [((inp(sh[:, k, 0]) * gmask[0] + inp(sh[:, k, 1]) * gmask[1]) + inp(sh[:, k, 2]) * gmask[2]) for k in range(nc)]
        ddx = ddy = ddz = zero
        if D > 0:
            B[1], B[2], B[3] = -C1 * y, C1 * z, -C1 * x
            ddy = ddy + (-C1) * t[1]; ddz = ddz + C1 * t[2]; ddx = ddx + (-C1) * t[3]
            if D > 1:
                xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
                B[4], B[5], B[6] = C2[0] * xy, C2[1] * yz, C2[2] * ((2.0 * zz - xx) - yy)
                B[7], B[8] = C2[3] * xz, C2[4] * (xx - yy)
                ddx = ddx + C2[0] * y * t[4]; ddy = ddy + C2[0] * x * t[4]
                ddy = ddy + C2[1] * z * t[5]; ddz = ddz + C2[1] * y * t[5]
                ddx = ddx + C2[2] * (-2.0 * x) * t[6]; ddy = ddy + C2[2] * (-2.0 * y) * t[6]; ddz = ddz + C2[2] * (4.0 * z) * t[6]
                ddx = ddx + C2[3] * z * t[7]; ddz = ddz + C2[3] * x * t[7]
                ddx = ddx + C2[4] * (2.0 * x) * t[8]; ddy = ddy + C2[4] * (-2.0 * y) * t[8]
                if D > 2:
                    B[9], B[10] = C3[0] * y * (3.0 * xx - yy), C3[1] * xy * z
                    B[11], B[12] = C3[2] * y * ((4.0 * zz - xx) - yy), C3[3] * z * ((2.0 * zz - 3.0 * xx) - 3.0 * yy)
                    B[13], B[14], B[15] = C3[4] * x * ((4.0 * zz - xx) - yy), C3[5] * z * (xx - yy), C3[6] * x * (xx - 3.0 * yy)
                    ddx = ddx + C3[0] * 6.0 * xy * t[9]; ddy = ddy + C3[0] * (3.0 * xx - 3.0 * yy) * t[9]
                    ddx = ddx + C3[1] * yz * t[10]; ddy = ddy + C3[1] * xz * t[10]; ddz = ddz + C3[1] * xy * t[10]
                    ddx = ddx + C3[2] * (-2.0 * xy) * t[11]; ddy = ddy + C3[2] * ((4.0 * zz - xx) - 3.0 * yy) * t[11]
                    ddz = ddz + C3[2] * 8.0 * yz * t[11]
                    ddx = ddx + C3[3] * (-6.0 * xz) * t[12]; ddy = ddy + C3[3] * (-6.0 * yz) * t[12]
                    ddz = ddz + C3[3] * ((6.0 * zz - 3.0 * xx) - 3.0 * yy) * t[12]
                    ddx = ddx + C3[4] * ((4.0 * zz - 3.0 * xx) - yy) * t[13]; ddy = ddy + C3[4] * (-2.0 * xy) * t[13]
                    ddz = ddz + C3[4] * 8.0 * xz * t[13]
                    ddx = ddx + C3[5] * 2.0 * xz * t[14]; ddy = ddy + C3[5] * (-2.0 * yz) * t[14]; ddz = ddz + C3[5] * (xx - yy) * t[14]
                    ddx = ddx + C3[6] * (3.0 * xx - 3.0 * yy) * t[15]; ddy = ddy + C3[6] * (-6.0 * xy) * t[15]
        dotp = (x * ddx + y * ddy) + z * ddz
        if bug != "no_sh_dir":
            dm = [dm[0] + (ddx - x * dotp) / ln, dm[1] + (ddy - y * dotp) / ln, dm[2] + (ddz - z * dotp) / ln]
        out["dL_dsh"] = [B[k] * gmask[ch] if k < nc else zero for k in range(M) for ch in range(3)]
        out["dL_dcolors_sh"] = gmask
    out["dL_dmeans3D"] = dm

    if I["scales"] is not None:
        mod = I["mod"]
        q = [inp(I["rots"][:, k]) for k in range(4)]
        qr, qx, qy, qz = q
        R = [1.0 - 2.0 * (qy * qy + qz * qz), 2.0 * (qx * qy - qr * qz), 2.0 * (qx * qz + qr * qy),
             2.0 * (qx * qy + qr * qz), 1.0 - 2.0 * (qx * qx + qz * qz), 2.0 * (qy * qz - qr * qx),
             2.0 * (qx * qz - qr * qy), 2.0 * (qy * qz + qr * qx), 1.0 - 2.0 * (qx * qx + qy * qy)]
        sv = [mod * inp(I["scales"][:, k]) for k in range(3)]
        Mx = [R[3 * r + cc] * sv[cc] for r in range(3) for cc in range(3)]
        dS = [g6[0], 0.5 * g6[1], 0.5 * g6[2], 0.5 * g6[1], g6[3], 0.5 * g6[4], 0.5 * g6[2], 0.5 * g6[4], g6[5]]
        dR, dsc = [None] * 9, []
        for cc in range(3):
            acc = zero
            for r in range(3):
                dMx = 2.0 * ((dS[3 * r] * Mx[cc] + dS[3 * r + 1] * Mx[3 + cc]) + dS[3 * r + 2] * Mx[6 + cc])
                acc = acc + R[3 * r + cc] * dMx
                dR[3 * r + cc] = dMx * sv[cc]
            dsc.append(acc * mod)
        t2 = qy * dR[2]
        first = (-qz * dR[1] - t2) if bug == "drot_sign" else (-qz * dR[1] + t2)
        out["dL_dscales"] = dsc
        out["dL_drotations"] = [
            2.0 * ((((first + qz * dR[3]) - qx * dR[5]) - qy * dR[6]) + qx * dR[7]),
            2.0 * ((((-2.0 * qx) * (dR[4] + dR[8]) + qy * (dR[1] + dR[3])) + qz * (dR[2] + dR[6])) + qr * (dR[7] - dR[5])),
            2.0 * ((((-2.0 * qy) * (dR[0] + dR[8]) + qx * (dR[1] + dR[3])) + qr * (dR[2] - dR[6])) + qz * (dR[5] + dR[7])),
            2.0 * ((((-2.0 * qz) * (dR[0] + dR[4]) + qr * (dR[3] - dR[1])) + qx * (dR[2] + dR[6])) + qy * (dR[5] + dR[7]))]
    return out, dec


SHAPES = dict(dL_dmeans3D=(3,), dL_dscales=(3,), dL_drotations=(4,), dL_dcov3D=(6,), dL_dopacity=(1,),
              dL_dcolors_precomp=(3,), dL_dcolors_sh=(3,), dL_dmeans2D=(3,))


def _inputs(st, dgeom):
    s, inp = st.settings, st.inputs
    vis = np.asarray(st.radii) > 0
    sel = lambda a: None if a is None else np.asarray(a)[vis]
    shs = inp["shs"]
    f = lambda c: f32(np.float32(c))
    return vis, dict(
        P=int(vis.sum()), view=np.asarray(s.viewmatrix, np.float32).reshape(16), proj=np.asarray(s.projmatrix, np.float32).reshape(16),
        campos=np.asarray(s.campos, np.float32).reshape(3), tanfovx=s.tanfovx, tanfovy=s.tanfovy,
        focal_x=f(np.float32(s.image_width) / (np.float32(2.0) * np.float32(s.tanfovx))),
        focal_y=f(np.float32(s.image_height) / (np.float32(2.0) * np.float32(s.tanfovy))),
        mod=f(s.scale_modifier), antialiasing=bool(s.antialiasing), D=int(s.sh_degree), M=int(st.cs.M),
        means=sel(inp["means3D"]), cov6=sel(st.cov3Ds), opac=sel(np.asarray(inp["opacities"]).reshape(-1)),
        scales=sel(inp["scales"]), rots=sel(inp["rotations"]), shs=sel(shs),
        clamped=np.asarray(st.clamped)[vis], dgeom=np.asarray(dgeom)[vis, :10])


def _pack(X, out, vis, I):
    """Outputs of _evaluate -> full [P, ...] arrays keyed like raster.preprocess_backward (zeros for culled Gaussians)."""
    P = vis.shape[0]
    res, bnd = {}, {}
    for k, lst in out.items():
        v = np.stack([np.broadcast_to(X.val(e), (I["P"],)) for e in lst], 1) if lst else np.zeros((I["P"], 0))
        b = np.stack([np.broadcast_to(X.bnd(e), (I["P"],)) for e in lst], 1) if lst else np.zeros((I["P"], 0))
        shape = (P, I["M"], 3) if k == "dL_dsh" else (P,) + SHAPES[k]
        fv, fb = np.zeros((P, v.shape[1])), np.zeros((P, v.shape[1]))
        fv[vis], fb[vis] = v, b
        res[k], bnd[k] = fv.reshape(shape), fb.reshape(shape)
    return res, bnd


def _copies(st, dgeom, vis, res, bnd):
    """The record's pass-through outputs: exact copies, budget 0."""
    P = vis.shape[0]
    g = np.asarray(dgeom, np.float64)
    m2 = np.zeros((P, 3)); m2[vis, :2] = g[vis, 0:2]
    res["dL_dmeans2D"], bnd["dL_dmeans2D"] = m2, np.zeros((P, 3))
    if st.inputs["colors_precomp"] is not None:
        cp = np.zeros((P, 3)); cp[vis] = g[vis, 6:9]
        res["dL_dcolors_precomp"], bnd["dL_dcolors_precomp"] = cp, np.zeros((P, 3))


def preprocess_backward64(st, dgeom, det2_eps=EPS_W):
    """float64 reference of the preprocess backward on the fp32 forward state `st` (oracle.raster.ForwardState) and the
    per-Gaussian record `dgeom` [P,>=10] (mean2D x/y, conic xx/xy/yy, opacity, rgb, inverse depth).  Returns
    dict(ref64=..., budget=..., ambiguous=[P] bool); ref64 and budget are dicts keyed like raster.preprocess_backward
    (dL_dmeans3D, dL_dscales, dL_drotations, dL_dcov3D, dL_dopacity [P,1], dL_dsh [P,M,3], dL_dcolors_precomp, and the
    factored dL_dcolors_sh), plus dL_dmeans2D [P,3].  `det2_eps` = 0 removes the upstream's +1e-7 on det^2 (for a
    comparison with the true derivative)."""
    vis, I = _inputs(st, dgeom)
    out, dec = _evaluate(_E64, I, det2_eps=det2_eps)
    ref, bud = _pack(_E64, out, vis, I)
    amb = np.zeros(I["P"], bool)
    extra = {k: np.zeros_like(v) for k, v in bud.items()}
    for name, (d, a) in dec.items():
        if not a.any():
            continue
        amb |= a
        fo, _ = _evaluate(_E64, I, force={name: np.where(a, ~d, d)}, det2_eps=det2_eps)
        r2, b2 = _pack(_E64, fo, vis, I)
        for k in bud:
            extra[k] += np.abs(r2[k] - ref[k]) + np.maximum(b2[k] - bud[k], 0.0)
    for k in bud:
        bud[k] = bud[k] + extra[k]
    _copies(st, dgeom, vis, ref, bud)
    ambiguous = np.zeros(vis.shape[0], bool)
    ambiguous[vis] = amb
    return dict(ref64=ref, budget=bud, ambiguous=ambiguous)


def preprocess_backward_f32(st, dgeom, bug=None):
    """A plain fp32 evaluation of the same expression tree, optionally with one planted bug (BUGS): a model of a kernel
    for the tests that show what the budget can and cannot see."""
    vis, I = _inputs(st, dgeom)
    out, _ = _evaluate(_F32, I, bug=bug)
    res, _ = _pack(_F32, out, vis, I)
    _copies(st, dgeom, vis, res, {})
    return res
