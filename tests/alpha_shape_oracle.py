"""Float64 references for gms_b200.alpha_shape (test-only).

alpha_faces: open3d's CreateFromPointCloudAlphaShape restated on scipy's Qhull Delaunay: every tetrahedron with
circumradius r = sqrt(Dx^2 + Dy^2 + Dz^2 - 4ac) / (2|a|) <= alpha pushes its four faces with ascending vertex indices, and
the faces pushed exactly once are kept.  Exact duplicate points are removed first (lowest index kept), as Qhull keeps one.
Returns a set of (a, b, c) original-index triples, and the tetrahedra's r - alpha for counting near-threshold decisions.

face_margins: the local rule of csrc/gms_alpha.cuh for given faces, brute force: the distances of each decision
(r_f - alpha, |T+| - beta, |T-| - beta, T+ - T-) from its threshold, for explaining a difference.

normals: KDTree k-nearest within radius (cKDTree, k = max_nn, distance_upper_bound = radius), float64 covariance and eigh,
with the sign rule of include/gms_b200.h; also the gap between the two smallest eigenvalues."""
from __future__ import annotations

import numpy as np


def dedup(P: np.ndarray):
    """(kept original indices ascending, the unique points) with exact duplicates collapsed to the lowest index."""
    _, first = np.unique(P, axis=0, return_index=True)
    keep = np.sort(first)
    return keep, P[keep]


def circumradius(v: np.ndarray) -> np.ndarray:
    """open3d's circumradius of tetrahedra v [T,4,3] from the 4x4 determinants."""
    sq = (v * v).sum(-1)
    one = np.ones(sq.shape)
    x, y, z = v[..., 0], v[..., 1], v[..., 2]
    det = lambda *cols: np.linalg.det(np.stack(cols, -1))
    a = det(x, y, z, one)
    c = det(sq, x, y, z)
    dx = det(sq, y, z, one)
    dy = det(sq, x, z, one)
    dz = det(sq, x, y, one)
    return np.sqrt(np.maximum(dx * dx + dy * dy + dz * dz - 4 * a * c, 0.0)) / (2 * np.abs(a))


def alpha_faces(P: np.ndarray, alpha: float):
    from scipy.spatial import Delaunay
    P = np.asarray(P, dtype=np.float64)
    keep, U = dedup(P)
    if len(U) < 4:
        return set(), np.zeros(0)
    try:
        T = Delaunay(U).simplices
    except Exception:           # all points coplanar: Qhull finds no tetrahedron
        return set(), np.zeros(0)
    r = circumradius(U[T])
    kept = np.sort(keep[T[r <= alpha]], axis=1)
    faces = np.concatenate([kept[:, [0, 1, 2]], kept[:, [0, 1, 3]], kept[:, [0, 2, 3]], kept[:, [1, 2, 3]]])
    if len(faces) == 0:
        return set(), r - alpha
    uniq, cnt = np.unique(faces, axis=0, return_counts=True)
    return {tuple(int(i) for i in f) for f in uniq[cnt == 1]}, r - alpha


def face_margins(P: np.ndarray, faces, alpha: float) -> np.ndarray:
    """For each face (a, b, c): the smallest distance of its decisions from their thresholds (0 when exactly on one)."""
    P = np.asarray(P, dtype=np.float64)
    keep, _ = dedup(P)
    live = np.zeros(len(P), bool)
    live[keep] = True
    out = []
    for a, b, c in faces:
        A = P[a]
        u, v = P[b] - A, P[c] - A
        w = np.cross(u, v)
        w2 = w @ w
        if w2 == 0:
            out.append(0.0)
            continue
        cf = (u @ u * np.cross(v, w) + v @ v * np.cross(w, u)) / (2 * w2)
        rf = np.sqrt(cf @ cf)
        m = [abs(rf - alpha) / alpha]
        if rf <= alpha:
            n = w / np.sqrt(w2)
            beta = np.sqrt(alpha * alpha - rf * rf)
            Q = P[live] - A - cf
            idx = np.nonzero(live)[0]
            sel = (idx != a) & (idx != b) & (idx != c)
            Q = Q[sel]
            s = Q @ n
            t = ((Q * Q).sum(1) - rf * rf) / (2 * np.where(s == 0, 1, s))
            tp = t[s > 0].min() if (s > 0).any() else np.inf
            tm = t[s < 0].max() if (s < 0).any() else -np.inf
            for T in (tp, tm):
                if np.isfinite(T):
                    m.append(abs(abs(T) - beta) / alpha)
            if np.isfinite(tp) and np.isfinite(tm):
                m.append(abs(tp - tm) / alpha)
        out.append(min(m))
    return np.asarray(out)


def normals(P: np.ndarray, radius: float = 0.1, max_nn: int = 30):
    """(normals [P,3] float64, eigen-gap [P] = lambda_1 - lambda_0 relative to the trace, neighbour count [P])."""
    from scipy.spatial import cKDTree
    P = np.asarray(P, dtype=np.float64)
    N = len(P)
    d, idx = cKDTree(P).query(P, k=max_nn, distance_upper_bound=radius)
    d = d.reshape(N, -1)
    idx = idx.reshape(N, -1)
    mean = P.mean(0)
    out = np.tile(np.array([0.0, 0.0, 1.0]), (N, 1))
    gap = np.full(N, np.inf)
    cnt = np.isfinite(d).sum(1)
    for i in range(N):
        if cnt[i] < 3:
            continue
        Q = P[idx[i, :cnt[i]]]
        C = np.cov(Q.T, bias=True)
        lam, V = np.linalg.eigh(C)
        n = V[:, 0]
        s = n @ (P[i] - mean)
        if s < 0 or (s == 0 and n[np.argmax(np.abs(n))] < 0):
            n = -n
        out[i] = n
        gap[i] = (lam[1] - lam[0]) / max(lam.sum(), 1e-300)
    return out, gap, cnt
