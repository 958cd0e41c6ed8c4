"""CPU-only: the two paths of tests/knn_oracle.py (all pairs, and k-d tree candidate sets with their brute-force fallback) give
the same bits at 20k points, uniform, clustered and with duplicates, and restate the definition on hand-checkable clouds."""
import numpy as np
import pytest

import knn_oracle as K


def _clouds():
    rng = np.random.default_rng(11)
    uniform = rng.uniform(-1.3, 1.3, (20_000, 3)).astype(np.float32)
    centres = rng.uniform(-1, 1, (40, 3))
    clustered = (centres[rng.integers(0, 40, 20_000)] + 0.002 * rng.standard_normal((20_000, 3))).astype(np.float32)
    half = rng.uniform(-1, 1, (10_000, 3)).astype(np.float32)
    dups = np.concatenate([half, half[rng.permutation(10_000)]])
    many = np.repeat(rng.uniform(-1, 1, (1000, 3)).astype(np.float32), 20, axis=0)   # 20 copies: every row falls back
    return {"uniform": uniform, "clustered": clustered, "duplicates": dups, "twenty_copies": many}


@pytest.mark.parametrize("name", ["uniform", "clustered", "duplicates", "twenty_copies"])
def test_candidate_path_equals_brute_force_bit_for_bit(name):
    pts = _clouds()[name]
    a = K.brute(pts)
    b, fallbacks = K.dist2(pts, return_fallbacks=True)
    assert a.dtype == b.dtype == np.float32
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    if name == "twenty_copies":
        assert fallbacks == pts.shape[0] and (a == 0).all()


def test_definition_on_small_clouds():
    # a unit square in the plane z = 0 plus its centre: corners see two edges (1) and the centre (0.5)
    pts = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [0.5, 0.5, 0]], np.float32)
    d = K.brute(pts)
    assert d[4] == np.float32((np.float32(0.5) + np.float32(0.5)) + np.float32(0.5)) / np.float32(3)
    assert (d[:4] == np.float32((np.float32(0.5) + np.float32(1)) + np.float32(1)) / np.float32(3)).all()
    # duplicates count separately: two copies of a point see each other at 0
    pts = np.array([[0, 0, 0], [0, 0, 0], [0, 0, 0], [2, 0, 0]], np.float32)
    assert (K.brute(pts)[:3] == np.float32(4) / np.float32(3)).all()
    assert K.brute(pts)[3] == np.float32(4)
    # the sum is float32 and rounded per operation, in the order ((dx*dx + dy*dy) + dz*dz)
    q = np.array([[0.1, 0.2, 0.3]], np.float32)
    p = np.array([[0.7, -0.4, 1.9]], np.float32)
    dx, dy, dz = (q - p)[0]
    assert K._d(q, p)[0] == (dx * dx + dy * dy) + dz * dz
    with pytest.raises(ValueError):
        K.brute(pts[:3])
