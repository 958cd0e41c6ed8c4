"""numpy restatement of the mesh-driven pseudo-mesh (gms_expand.cuh gms_pm_*, k_pseudomesh_bind, k_pseudomesh_repose).

Every step is the product's own sequence of correctly rounded operations, in float32 where the product uses fp32 and in
float64 where it uses double; numpy performs each +, -, *, / and sqrt separately (no contraction), so each function agrees
with the kernels bit for bit.  The nearest face is a brute-force argmin over ALL faces (lowest index on an exact tie), with
degenerate faces excluded."""
import numpy as np

F32 = np.float32


def centroids(t):
    """t [N,3,3] float32 -> ((v0 + v1) + v2) / 3 [N,3] float32."""
    t = np.asarray(t, dtype=F32)
    return ((t[:, 0] + t[:, 1]) + t[:, 2]) / F32(3)


def _norm(x):
    return np.sqrt((x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2])


def frames(v1, v2, v3):
    """(n, e1, e2, degenerate) of faces given by their corners [N,3] float32."""
    v1, v2, v3 = (np.asarray(v, dtype=F32) for v in (v1, v2, v3))
    a, b = v2 - v1, v3 - v1
    c = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                  a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    la, lb, lc = _norm(a), _norm(b), _norm(c)
    with np.errstate(divide="ignore", invalid="ignore"):
        n, e1, e2 = c / lc[:, None], a / la[:, None], b / lb[:, None]
    return n, e1, e2, (la == 0) | (lb == 0) | (lc == 0)


def distances(q, c):
    """Squared distances [Nq,Nc] in float64, (dx*dx + dy*dy) + dz*dz."""
    q, c = np.asarray(q, dtype=np.float64), np.asarray(c, dtype=np.float64)
    d = [q[:, None, k] - c[None, :, k] for k in range(3)]
    return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def _dot(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def coefficients(n, e1, e2, v1, w):
    """[n|e1|e2] c_j = w_j - v1 solved in float64 through the adjugate, rounded to float32: [P,3,3]."""
    n, e1, e2 = (np.asarray(x, dtype=np.float64) for x in (n, e1, e2))
    r = [_cross(e1, e2), _cross(e2, n), _cross(n, e1)]
    det = _dot(n, r[0])
    out = np.empty((n.shape[0], 3, 3), dtype=F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        for j in range(3):
            d = np.asarray(w[:, j], dtype=np.float64) - np.asarray(v1, dtype=np.float64)
            for k in range(3):
                out[:, j, k] = (_dot(d, r[k]) / det).astype(F32)
    return out


def bind(triangles, vertices, faces, chunk=1024):
    """(face int64 [P], coeffs float32 [P,3,3], n_degenerate, best and second-best distance [P,2]) of a pseudo-mesh
    bound to a mesh.  ValueError when every face is degenerate."""
    tri = np.asarray(triangles, dtype=F32)
    fv = np.asarray(vertices, dtype=F32)[np.asarray(faces)]
    n, e1, e2, deg = frames(fv[:, 0], fv[:, 1], fv[:, 2])
    if deg.all():
        raise ValueError("every face is degenerate")
    cf, q = centroids(fv), centroids(tri)
    P = tri.shape[0]
    idx = np.zeros(P, dtype=np.int64)
    best2 = np.zeros((P, 2))
    for s in range(0, P, chunk):
        d = distances(q[s:s + chunk], cf)
        d[:, deg] = np.inf
        idx[s:s + chunk] = np.argmin(d, axis=1)
        best2[s:s + chunk] = np.sort(d, axis=1)[:, :2] if d.shape[1] > 1 else np.concatenate([d, d], 1)
    coeffs = coefficients(n[idx], e1[idx], e2[idx], fv[idx, 0], tri)
    return idx, coeffs, int(deg.sum()), best2


def repose(face, coeffs, vertices, faces):
    """Triangles [P,3,3] float32: w_j = ((v1 + c_j0 n) + c_j1 e1) + c_j2 e2 in the pose `vertices`."""
    fv = np.asarray(vertices, dtype=F32)[np.asarray(faces)[np.asarray(face)]]
    n, e1, e2, _ = frames(fv[:, 0], fv[:, 1], fv[:, 2])
    c = np.asarray(coeffs, dtype=F32)
    v1 = fv[:, 0]
    out = np.empty_like(c)
    for j in range(3):
        out[:, j] = ((v1 + c[:, j, 0:1] * n) + c[:, j, 1:2] * e1) + c[:, j, 2:3] * e2
    return out


def condition_numbers(n, e1, e2):
    """2-norm condition number of every [n|e1|e2]."""
    A = np.stack([np.asarray(x, dtype=np.float64) for x in (n, e1, e2)], 2)
    return np.linalg.cond(A)
