"""CPU-only checks of the mesh-driven pseudo-mesh edit.

1. The numpy oracle (pseudomesh_oracle.py) reproduces the reference's own edit (pseudomesh_edit.npz, generated from
   scripts/edit_pseudomesh_based_on_estimated_mesh.py): every nearest-face index, and the coefficients and edited triangles
   within a tolerance scaled by each frame's condition number.
2. The product's device functions (gms_expand.cuh gms_pm_*), compiled for the CPU with g++, agree with the oracle bit for
   bit and with a float64 restatement of the same arithmetic within fp32 rounding.
3. io_obj reads and writes the OBJ subset the workflow uses."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import pseudomesh_oracle as orc
from gms_b200 import io_obj

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gaussian-mesh-splatting_b200", "csrc")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "pseudomesh_edit.npz"))


def test_oracle_binds_like_the_reference_kd_tree(golden):
    idx, coeffs, n_deg, _ = orc.bind(golden["triangles"], golden["vertices"], golden["faces"])
    assert n_deg == 0 and golden["triangles"].shape[0] != 3
    np.testing.assert_array_equal(idx, golden["index_of_closest"])
    fv = golden["vertices"][golden["faces"][idx]]
    n, e1, e2, _ = orc.frames(fv[:, 0], fv[:, 1], fv[:, 2])
    cond = orc.condition_numbers(n, e1, e2)
    # the reference solves in fp32 (LU); the oracle in double: both are within ~cond * eps_fp32 of the exact solution
    scale = np.abs(golden["coeffs"]).max(axis=(1, 2))
    err = np.abs(coeffs - golden["coeffs"]).max(axis=(1, 2)) / (cond * np.maximum(scale, 1e-30) * np.finfo(np.float32).eps)
    print(f"[pseudomesh oracle] worst coefficient error {err.max():.3g} x cond x |c| x eps32 (cond up to {cond.max():.3g})")
    assert err.max() <= 16


def test_oracle_reposes_like_the_reference(golden):
    idx, coeffs, _, _ = orc.bind(golden["triangles"], golden["vertices"], golden["faces"])
    edited = orc.repose(idx, coeffs, golden["vertices_edited"], golden["faces"])
    fv = golden["vertices"][golden["faces"][idx]]
    cond = orc.condition_numbers(*orc.frames(fv[:, 0], fv[:, 1], fv[:, 2])[:3])
    extent = np.abs(golden["edited_triangles"]).max(axis=(1, 2)) + np.abs(coeffs).max(axis=(1, 2))
    err = np.abs(edited - golden["edited_triangles"]).max(axis=(1, 2)) / (cond * extent * np.finfo(np.float32).eps)
    print(f"[pseudomesh oracle] worst edited-triangle error {err.max():.3g} x cond x extent x eps32")
    assert err.max() <= 16


def test_oracle_repose_on_the_rest_pose_returns_the_pseudo_mesh(golden):
    idx, coeffs, _, _ = orc.bind(golden["triangles"], golden["vertices"], golden["faces"])
    back = orc.repose(idx, coeffs, golden["vertices"], golden["faces"])
    assert np.abs(back - golden["triangles"]).max() <= 1e-5


# ---- the device functions, compiled for the CPU
SHIM = r'''
#include "gms_expand.cuh"
extern "C" {
int pm_frame(const float* v, float* out) {      /* v: 9 floats; out: n, e1, e2 */
    GmsPmFrame f;
    const bool deg = gms_pm_frame(v, v + 3, v + 6, f);
    for (int k = 0; k < 3; k++) { out[k] = f.n[k]; out[3 + k] = f.e1[k]; out[6 + k] = f.e2[k]; }
    return deg;
}
void pm_centroid(const float* v, float* m) { gms_pm_centroid(v, v + 3, v + 6, m); }
double pm_dist2(const float* q, const float* c) { return gms_pm_dist2(q[0], q[1], q[2], c[0], c[1], c[2]); }
void pm_coeffs(const float* v, const float* w, float* c) {
    GmsPmFrame f;
    gms_pm_frame(v, v + 3, v + 6, f);
    gms_pm_coeffs(f, v, w, c);
}
void pm_repose(const float* v, const float* c, float* w) {
    GmsPmFrame f;
    gms_pm_frame(v, v + 3, v + 6, f);
    gms_pm_repose(f, v, c, w);
}
}
'''


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("pm_shim")
    src, so = d / "pm_shim.cpp", d / "libpm_shim.so"
    src.write_text(SHIM)
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-I", CSRC,
                           str(src), "-o", str(so)])
    L = C.CDLL(str(so))
    L.pm_frame.restype = C.c_int
    L.pm_dist2.restype = C.c_double
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _faces(n, seed):
    g = np.random.default_rng(seed)
    v = g.standard_normal((n, 3, 3)).astype(np.float32)
    v[:, 1:] = v[:, :1] + (10.0 ** g.uniform(-3, 1, (n, 2, 1))) * g.standard_normal((n, 2, 3))
    v[0, 1] = v[0, 0]                         # zero edge
    v[1, 2] = v[1, 0] + 2 * (v[1, 1] - v[1, 0])     # collinear: zero cross product up to rounding
    v[2, 2] = v[2, 0]
    return v.astype(np.float32)


def test_device_functions_match_the_oracle_bit_for_bit(shim):
    faces = _faces(300, 1)
    g = np.random.default_rng(2)
    w = (faces[:, :1] + g.standard_normal((300, 3, 3)) * 0.3).astype(np.float32)
    n, e1, e2, deg = orc.frames(faces[:, 0], faces[:, 1], faces[:, 2])
    co = orc.coefficients(n, e1, e2, faces[:, 0], w)
    moved = (faces * np.float32(1.7) + np.float32(0.25)).astype(np.float32)
    cen = orc.centroids(faces)
    for i in range(300):
        fr = np.empty(9, np.float32)
        d = shim.pm_frame(_p(faces[i]), _p(fr))
        assert bool(d) == bool(deg[i]), i
        np.testing.assert_array_equal(fr, np.concatenate([n[i], e1[i], e2[i]]))
        m = np.empty(3, np.float32)
        shim.pm_centroid(_p(faces[i]), _p(m))
        np.testing.assert_array_equal(m, cen[i])
        assert shim.pm_dist2(_p(cen[i]), _p(cen[(i + 1) % 300])) == orc.distances(cen[i:i + 1], cen[(i + 1) % 300:][:1])[0, 0]
        if deg[i]:
            continue
        c = np.empty(9, np.float32)
        shim.pm_coeffs(_p(faces[i]), _p(np.ascontiguousarray(w[i])), _p(c))
        np.testing.assert_array_equal(c.reshape(3, 3), co[i])
        out = np.empty(9, np.float32)
        shim.pm_repose(_p(moved[i]), _p(c), _p(out))
        want = orc.repose(np.array([0]), co[i:i + 1], moved[i], np.array([[0, 1, 2]]))[0]
        np.testing.assert_array_equal(out.reshape(3, 3), want)
    assert deg[:3].all() and not deg[3:].any()


def test_device_functions_match_a_float64_restatement(shim):
    """The frame, the solve and the re-pose against the same formulas in float64 (numpy.linalg.solve for the system)."""
    faces = _faces(300, 3)[3:]
    g = np.random.default_rng(4)
    w = (faces[:, :1] + g.standard_normal((faces.shape[0], 3, 3)) * 0.3).astype(np.float32)
    worst = 0.0
    for i in range(faces.shape[0]):
        v = faces[i].astype(np.float64)
        a, b = v[1] - v[0], v[2] - v[0]
        F = np.stack([np.cross(a, b) / np.linalg.norm(np.cross(a, b)), a / np.linalg.norm(a), b / np.linalg.norm(b)], 1)
        fr = np.empty(9, np.float32)
        shim.pm_frame(_p(faces[i]), _p(fr))
        sin_inv = np.linalg.norm(a) * np.linalg.norm(b) / np.linalg.norm(np.cross(a, b))   # the cross product's cancellation
        err = np.abs(fr.reshape(3, 3).T - F)
        assert err[:, 0].max() <= 4 * sin_inv * np.finfo(np.float32).eps and err[:, 1:].max() <= 2 * np.finfo(np.float32).eps
        c = np.empty(9, np.float32)
        shim.pm_coeffs(_p(faces[i]), _p(np.ascontiguousarray(w[i])), _p(c))
        A = fr.reshape(3, 3).T.astype(np.float64)         # the fp32 frame, columns n, e1, e2
        want = np.linalg.solve(A, (w[i].astype(np.float64) - v[0]).T).T
        kappa = np.linalg.cond(A)
        err = np.abs(c.reshape(3, 3) - want).max() / (np.abs(want).max() * np.finfo(np.float32).eps * (1 + kappa * 1e-7))
        worst = max(worst, err)
        out = np.empty(9, np.float32)
        shim.pm_repose(_p(faces[i]), _p(c), _p(out))
        ext = np.abs(w[i]).max() + np.abs(c).max()
        assert np.abs(out.reshape(3, 3) - w[i]).max() <= 8 * kappa * ext * np.finfo(np.float32).eps, i
    print(f"[pseudomesh shim] worst coefficient error {worst:.3g} ulp-scale")
    assert worst <= 1.0


# ---- io_obj
def test_obj_round_trip(tmp_path):
    g = torch.Generator().manual_seed(0)
    v = torch.randn(20, 3, generator=g)
    f = torch.randint(0, 20, (30, 3), generator=g)
    path = str(tmp_path / "m.obj")
    io_obj.write_obj(path, v, f)
    text = open(path).read().splitlines()
    assert text[0] == "v %f %f %f" % tuple(v[0].tolist()) and text[20] == "f %d %d %d" % tuple((f[0] + 1).tolist())
    v2, f2 = io_obj.read_obj(path)
    assert v2.dtype == torch.float32 and f2.dtype == torch.int64
    assert torch.equal(f2, f) and float((v2 - v).abs().max()) <= 5e-7


def test_obj_slash_negative_index_and_polygon_forms(tmp_path):
    path = tmp_path / "q.obj"
    path.write_text("# comment\nmtllib x.mtl\no thing\nv 0 0 0\nv 1 0 0\nv 1 1 0 1.0\nv 0 1 0\nvt 0 0\nvn 0 0 1\n"
                    "usemtl m\ns off\nf 1/1/1 2/1/1 3/1/1 4/1/1\nf -4//1 -2//1 -1//1\nf 1/1 3/1 4/1\nv 0 0 1\n"
                    "f 5 1 2 3 4\n")
    v, f = io_obj.read_obj(str(path))
    assert v.shape == (5, 3) and float(v[2, 1]) == 1.0
    assert f.tolist() == [[0, 1, 2], [0, 2, 3], [0, 2, 3], [0, 2, 3], [4, 0, 1], [4, 1, 2], [4, 2, 3]]


def test_obj_triangle_soup_and_bad_indices(tmp_path):
    tri = torch.arange(27, dtype=torch.float32).reshape(3, 3, 3)
    path = str(tmp_path / "soup.obj")
    io_obj.write_obj(path, *io_obj.triangle_soup(tri))
    v, f = io_obj.read_obj(path)
    assert torch.equal(v[f], tri)
    bad = tmp_path / "bad.obj"
    bad.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 4\n")
    with pytest.raises(ValueError):
        io_obj.read_obj(str(bad))
    bad.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 0 1 2\n")
    with pytest.raises(ValueError):
        io_obj.read_obj(str(bad))
