"""numpy float32 restatement of gms_knn_dist2 (include/gms_b200.h): for every point, ((b0 + b1) + b2) / 3 of the three
smallest d(q,p) = (dx*dx + dy*dy) + dz*dz over the other points, every operation one round-to-nearest float32 op (numpy never
contracts into an FMA).

Two paths give the same bits:
  brute(points)   every pair, in chunks of rows (P up to ~20k);
  dist2(points)   for large P: candidate sets from scipy's cKDTree (k = 16, float64), each candidate's float32 d recomputed.
                  A row whose 16th float64 squared distance is not clearly above its float32 b2 falls back to brute force.
Why the candidate set holds the answer: every point outside it has an exact squared distance >= D16 (the 16th float64
distance, squared; float32 coordinates are exact in float64).  Its float32 d has a relative error below 6u (u = 2^-24: three
rounded differences, three products, two sums), so d >= D16 (1 - 6u).  With D16 (1 - 1e-5) > b2 every such point has d > b2
and cannot be among the three smallest values.  Rows near underflow (D16 <= 1e-30) fall back as well."""
from __future__ import annotations

import numpy as np

K_CAND = 16
MARGIN = 1e-5
TINY = 1e-30


def _d(q: np.ndarray, p: np.ndarray) -> np.ndarray:
    """q [..., 3], p [..., 3] float32 -> (dx*dx + dy*dy) + dz*dz in float32."""
    dx, dy, dz = q[..., 0] - p[..., 0], q[..., 1] - p[..., 1], q[..., 2] - p[..., 2]
    return (dx * dx + dy * dy) + dz * dz


def _finish(best3: np.ndarray) -> np.ndarray:
    b = np.sort(best3, axis=1)
    return ((b[:, 0] + b[:, 1]) + b[:, 2]) / np.float32(3)


def _brute_rows(pts: np.ndarray, rows: np.ndarray, chunk: int) -> np.ndarray:
    out = np.empty((rows.shape[0], 3), np.float32)
    for s in range(0, rows.shape[0], chunk):
        r = rows[s:s + chunk]
        d = _d(pts[r][:, None, :], pts[None, :, :])
        d[np.arange(r.shape[0]), r] = np.inf
        out[s:s + chunk] = np.partition(d, 2, axis=1)[:, :3]
    return out


def brute(points, chunk: int = 256) -> np.ndarray:
    pts = np.ascontiguousarray(points, dtype=np.float32)
    if pts.shape[0] < 4:
        raise ValueError("need P >= 4")
    return _finish(_brute_rows(pts, np.arange(pts.shape[0]), chunk))


def dist2(points, chunk: int = 256, return_fallbacks: bool = False):
    """Same bits as brute(), by candidate sets; with return_fallbacks, also the number of rows that fell back to brute force."""
    from scipy.spatial import cKDTree
    pts = np.ascontiguousarray(points, dtype=np.float32)
    P = pts.shape[0]
    if P < 4:
        raise ValueError("need P >= 4")
    k = min(K_CAND, P)
    p64 = pts.astype(np.float64)
    D, I = cKDTree(p64).query(p64, k=k)
    d = _d(pts[:, None, :], pts[I])
    d[I == np.arange(P)[:, None]] = np.inf                  # the point itself (wherever the tree put it among ties)
    best = np.partition(d, 2, axis=1)[:, :3]
    b2 = best.max(axis=1).astype(np.float64)
    d16 = D[:, -1] ** 2
    bad = np.flatnonzero(~((d16 * (1 - MARGIN) > b2) & (d16 > TINY))) if k < P else np.empty(0, np.int64)
    if bad.size:
        best[bad] = _brute_rows(pts, bad, chunk)
    out = _finish(best)
    return (out, int(bad.size)) if return_fallbacks else out


def surface_points(n: int, seed: int = 0, faces: int = 20_000) -> np.ndarray:
    """n points sampled uniformly per face on scenes.object_mesh (a torus around a bumpy sphere): a clustered, COLMAP-like
    cloud on 2D surfaces, float32."""
    from gms_b200 import scenes
    v, f = scenes.object_mesh(faces)
    rng = np.random.default_rng(seed)
    fi = rng.integers(0, f.shape[0], n)
    r1, r2 = np.sqrt(rng.random(n)), rng.random(n)
    a, b, c = v[f[fi, 0]].astype(np.float64), v[f[fi, 1]].astype(np.float64), v[f[fi, 2]].astype(np.float64)
    return ((1 - r1)[:, None] * a + (r1 * (1 - r2))[:, None] * b + (r1 * r2)[:, None] * c).astype(np.float32)
