"""GPU: gms_b200.alpha_shape (gms_alpha_shape, gms_estimate_normals) against the float64 references of
tests/alpha_shape_oracle.py, and cli.create_dummy_mesh between cli.save_pseudomesh and cli.edit_pseudomesh.

Triangle sets are compared through original point indices.  A face in the symmetric difference must have a decision within
1e-9 alpha of its threshold (face_margins); the counts of such faces and of the oracle's near-threshold tetrahedra are
printed, and on these seeds are expected to be 0."""
import argparse
import os

import numpy as np
import pytest
import torch

import alpha_shape_cases as cases
import alpha_shape_oracle as oracle
from gms_b200 import _lib, io_obj
from gms_b200.alpha_shape import alpha_shape, estimate_normals
from gms_b200.cli import create_dummy_mesh, edit_pseudomesh, save_pseudomesh
from gms_b200.model import FreeGaussianModel

pytestmark = pytest.mark.gpu

MARGIN = 1e-9


def check_set(P32: np.ndarray, alpha: float, what: str):
    pts = torch.tensor(P32, device="cuda")
    v, f, idx = alpha_shape(pts, alpha)
    assert v.dtype == torch.float32 and f.dtype == torch.int64 and idx.dtype == torch.int64
    assert torch.equal(v, pts[idx]), "vertices must be points[index]"
    ih = idx.cpu().numpy()
    assert np.all(np.diff(ih) > 0), "index must be strictly ascending"
    fo = ih[f.cpu().numpy()] if len(f) else np.zeros((0, 3), np.int64)
    assert np.all(fo[:, 0] < fo[:, 1]) and np.all(fo[:, 1] < fo[:, 2]), "each face in ascending index order"
    assert [tuple(r) for r in fo.tolist()] == sorted(tuple(r) for r in fo.tolist()), "faces in lexicographic order"
    assert np.array_equal(np.unique(fo), ih), "vertices are exactly the referenced points"
    got = set(map(tuple, fo.tolist()))
    P64 = P32.astype(np.float64)
    ref, rmargin = oracle.alpha_faces(P64, alpha)
    diff = sorted(got ^ ref)
    margins = oracle.face_margins(P64, diff, alpha)
    near_tets = int((np.abs(rmargin) < MARGIN * alpha).sum())
    print(f"{what}: alpha {alpha}: {len(got)} faces, oracle {len(ref)}, differ {len(diff)}, "
          f"near-threshold tetrahedra {near_tets}, differing faces within {MARGIN} alpha of a threshold {int((margins < MARGIN).sum())}")
    assert np.all(margins < MARGIN), [(d, m) for d, m in zip(diff, margins) if m >= MARGIN][:10]
    return got


@pytest.mark.parametrize("alpha", [0.06, 0.1, 0.15])
def test_uniform_box(alpha):
    assert len(check_set(cases.box(3000, 5), alpha, "box")) > 0


@pytest.mark.parametrize("alpha", [0.08, 0.12, 0.2])
def test_noisy_sphere_shell(alpha):
    assert len(check_set(cases.shell(4000, 6), alpha, "shell")) > 0


def test_duplicated_points():
    base = cases.box(1500, 7)
    rng = np.random.default_rng(8)
    P = np.concatenate([base, base[rng.choice(1500, 400)]])
    P = P[rng.permutation(len(P))]
    got = check_set(P, 0.12, "duplicates")
    _, first = np.unique(P, axis=0, return_index=True)
    assert {i for t in got for i in t} <= set(first.tolist()), "only the lowest index of equal points is used"


@pytest.fixture(scope="module")
def soup():
    return cases.pseudomesh_points(20000, seed=3)         # 60k points: the x2 pseudo-mesh of 20k flat Gaussians


@pytest.mark.parametrize("alpha", [0.01, 0.02])       # at 0.003 this 60k-point soup is too sparse for any face
def test_pseudomesh_of_a_flat_model(soup, alpha):
    assert len(check_set(soup.cpu().numpy(), alpha, "pseudo-mesh")) > 0


def test_overflowing_lists_take_the_global_path():
    rng = np.random.default_rng(9)
    x = rng.standard_normal((700, 3))
    clump = x / np.linalg.norm(x, axis=1, keepdims=True) * 0.03 * rng.random((700, 1)) ** (1 / 3) + 2.0
    P = np.concatenate([cases.box(2000, 10), clump]).astype(np.float32)
    alpha = 0.025
    from scipy.spatial import cKDTree
    longest = max(len(l) - 1 for l in cKDTree(P.astype(np.float64)).query_ball_point(P.astype(np.float64), 3 * alpha))
    assert longest > _lib.ALPHA_LIST_CAP
    assert len(check_set(P, alpha, "overflow")) > 0


def check_normals(P32: np.ndarray, what: str, radius=0.1, max_nn=30):
    got = estimate_normals(torch.tensor(P32, device="cuda"), radius, max_nn).cpu().numpy().astype(np.float64)
    P64 = P32.astype(np.float64)
    ref, gap, cnt = oracle.normals(P64, radius, max_nn)
    assert np.allclose(np.linalg.norm(got, axis=1), 1, atol=1e-6)
    assert np.array_equal(got[cnt < 3], np.tile([0.0, 0.0, 1.0], ((cnt < 3).sum(), 1)))
    ok = (cnt >= 3) & (gap > 1e-6)
    sin = np.linalg.norm(np.cross(got[ok], ref[ok]), axis=1)
    tol = 1e-11 / gap[ok] + 3e-7
    print(f"{what}: {len(P32)} points, {(cnt < 3).sum()} with fewer than 3 neighbours, {(~ok & (cnt >= 3)).sum()} excluded "
          f"for a near-zero eigen-gap, largest sin {sin.max():.3g}")
    assert np.all(sin <= tol), (sin / tol).max()
    d = ((P64 - P64.mean(0)) * ref).sum(1)
    sure = ok & (np.abs(d) > 1e-6)
    assert np.all((got[sure] * ref[sure]).sum(1) > 0), "sign rule: n.(x - mean) >= 0"
    assert np.all(((P64 - P64.mean(0)) * got).sum(1)[sure] > 0)


def test_normals_shell():
    check_normals(cases.shell(4000, 11), "shell")


def test_normals_pseudomesh(soup):
    check_normals(soup.cpu().numpy(), "pseudo-mesh")


def test_deterministic(soup):
    a = alpha_shape(soup, 0.01)
    b = alpha_shape(soup, 0.01)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert torch.equal(estimate_normals(soup), estimate_normals(soup))


def test_refusals():
    pts = torch.zeros(5, 3, device="cuda")
    for bad in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(ValueError, match="alpha"):
            alpha_shape(pts, bad)
    with pytest.raises(ValueError, match="finite"):
        alpha_shape(torch.tensor([[0.0, 0.0, float("nan")]] * 4, device="cuda"), 0.1)
    with pytest.raises(ValueError, match="max_nn"):
        estimate_normals(pts, 0.1, 0)
    with pytest.raises(ValueError, match="radius"):
        estimate_normals(pts, 0.0)
    v, f, i = alpha_shape(torch.zeros(0, 3, device="cuda"), 0.1)
    assert v.shape == (0, 3) and f.shape == (0, 3) and i.shape == (0,)
    v, f, i = alpha_shape(pts[:3] + torch.arange(9.0, device="cuda").reshape(3, 3) ** 2, 100.0)
    assert f.shape == (0, 3)                              # three points have no tetrahedron
    import ctypes
    nf, nv = ctypes.c_int64(7), ctypes.c_int64(7)
    a = _lib.AlphaShapeArgs()
    a.P, a.points, a.alpha, a.n_faces, a.n_vertices = 4, pts.data_ptr(), -1.0, ctypes.pointer(nf), ctypes.pointer(nv)
    never = _lib.ALLOC_FN(lambda user, which, nbytes: 0)
    assert _lib.lib().gms_alpha_shape(ctypes.byref(a), never, None, None) == _lib.GMS_E_ARG
    assert (nf.value, nv.value) == (7, 7), "refused before touching the outputs"


def _flat_checkpoint(root: str, n: int) -> str:
    g = cases.surface_flat_gaussians(n, seed=12)
    out = os.path.join(root, "model")
    ply = os.path.join(out, "point_cloud", "iteration_7", "point_cloud.ply")
    os.makedirs(os.path.dirname(ply))
    FreeGaussianModel(g["xyz"], g["scaling"], g["rotation"], torch.cat([g["features_dc"], g["features_rest"]], 1).contiguous(),
                      g["opacity"], "gs_flat", "cuda", 3).save(ply)
    with open(os.path.join(out, "cfg_args"), "w") as fh:
        fh.write(str(argparse.Namespace(sh_degree=3, model_path=out, gs_type="gs_flat")))
    return out


def test_cli_save_create_edit(tmp_path, capsys):
    out = _flat_checkpoint(str(tmp_path), 3000)
    save_pseudomesh.main(["--model_path", out])
    d = os.path.join(out, "pseudomesh_info", "ours_7")
    tri_path = os.path.join(d, "triangles.pt")
    res = create_dummy_mesh.main(["--pseudomesh_path", tri_path, "--alpha", "0.02"])
    mesh = os.path.join(d, "mesh_alpha_0_003.obj")
    assert res["path"] == mesh and os.path.exists(mesh) and res["faces"] > 0
    tri = torch.load(tri_path)
    pts = (tri.reshape(-1, 3) * 2).float()
    v_want, f_want, idx = alpha_shape(pts, 0.02)
    want = tmp_path / "want.obj"
    io_obj.write_obj(str(want), v_want, f_want, estimate_normals(pts)[idx])
    assert open(mesh, "rb").read() == want.read_bytes()
    v, f = io_obj.read_obj(mesh)
    assert f.shape[0] == res["faces"] and v.shape[0] == res["vertices"]
    edited = tmp_path / "edited.obj"
    io_obj.write_obj(str(edited), v + torch.tensor([0.1, 0.0, -0.05]), f)
    r = edit_pseudomesh.main(["--triangle_soup_path", os.path.join(d, "scale_2.obj"), "--mesh_path", mesh, "--edited_mesh_path",
                              str(edited), "--save_dir", str(tmp_path / "edit"), "--scale", "2"])
    assert r["degenerate_faces"] == 0 and r["triangles"] == tri.shape[0]
    # an alpha below every circumradius: an empty OBJ and a message
    res = create_dummy_mesh.main(["--pseudomesh_path", tri_path, "--alpha", "1e-9"])
    assert res["faces"] == 0 and open(mesh).read() == ""
    assert "No tetrahedron" in capsys.readouterr().out
