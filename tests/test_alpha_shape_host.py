"""CPU-only checks of the dummy-mesh path (gms_b200.alpha_shape, cli.create_dummy_mesh):
- the Qhull oracle (tests/alpha_shape_oracle.py) on hand-built cases;
- the product's float64 face predicates and eigen-solver (csrc/gms_alpha.cuh built for the CPU) against that oracle;
- the ctypes mirrors of the two argument structs, the CLI parser against the script's, the output name, and write_obj with
  normals."""
import ctypes
import itertools
import os
import subprocess

import numpy as np
import pytest
import torch

import alpha_shape_oracle as oracle
from gms_b200 import _lib, io_obj
from gms_b200.cli import create_dummy_mesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

TET = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], dtype=np.float64) * 0.1     # circumradius 0.1 * sqrt(3)
R_TET = 0.1 * np.sqrt(3)


def _faces(*tris):
    return {tuple(sorted(t)) for t in tris}


# ---- the oracle on hand-built cases

def test_oracle_regular_tetrahedron():
    assert oracle.alpha_faces(TET, R_TET * 1.01)[0] == set(itertools.combinations(range(4), 3))
    assert oracle.alpha_faces(TET, R_TET * 0.99)[0] == set()


def test_oracle_two_tetrahedra_drop_the_shared_face():
    P = np.vstack([TET, [[1.0, 1.0, -1.0]]]) * 1.0
    P[4] = [0.12, 0.12, -0.12]                      # beyond face (0, 1, 2), on the far side from vertex 3
    faces, _ = oracle.alpha_faces(P, 1.0)
    assert len(faces) == 6
    assert (0, 1, 2) not in faces
    assert faces == _faces((0, 1, 3), (0, 2, 3), (1, 2, 3), (0, 1, 4), (0, 2, 4), (1, 2, 4))


def test_oracle_octahedron():
    P = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], dtype=np.float64)
    faces, r = oracle.alpha_faces(P, 1.0 + 1e-9)
    assert len(r) == 4                              # Qhull splits it into four tetrahedra around one diagonal
    octa = {tuple(sorted((x, y, z))) for x in (0, 1) for y in (2, 3) for z in (4, 5)}
    assert faces == octa                            # the eight outer faces; the inner ones are shared and dropped
    assert oracle.alpha_faces(P, 0.99)[0] == set()


def test_oracle_duplicates_keep_the_lowest_index():
    P = np.vstack([TET, TET[[2, 0]]])               # indices 4, 5 repeat 2 and 0
    assert oracle.alpha_faces(P, 1.0)[0] == set(itertools.combinations(range(4), 3))
    Q = np.vstack([TET[[1]], TET])                  # index 2 repeats index 0's point: the lowest copy, 0, stays
    assert oracle.alpha_faces(Q, 1.0)[0] == _faces((0, 1, 3), (0, 1, 4), (0, 3, 4), (1, 3, 4))


def test_oracle_fewer_than_four_points():
    for n in range(4):
        assert oracle.alpha_faces(TET[:n], 1.0)[0] == set()


# ---- the product's predicates, built for the CPU

@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("alpha_shim") / "libalpha_shim.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(HERE, "hostshim", "alpha_shim.cpp")])
    L = ctypes.CDLL(out)
    L.shim_alpha_faces.restype = ctypes.c_int64
    L.shim_alpha_faces.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_double, ctypes.c_void_p, ctypes.c_int64]
    L.shim_min_eigvec.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return L


def shim_faces(L, P32: np.ndarray, alpha: float):
    P32 = np.ascontiguousarray(P32, dtype=np.float32)
    n = L.shim_alpha_faces(len(P32), P32.ctypes.data, alpha, None, 0)
    out = np.zeros((max(n, 1), 3), dtype=np.int64)
    L.shim_alpha_faces(len(P32), P32.ctypes.data, alpha, out.ctypes.data, n)
    return out[:n]


def clouds():
    rng = np.random.default_rng(0)
    box = rng.random((300, 3)).astype(np.float32)
    x = rng.standard_normal((400, 3))
    shell = (x / np.linalg.norm(x, axis=1, keepdims=True) * (1 + 0.02 * rng.standard_normal((400, 1)))).astype(np.float32)
    return [("box", box, 0.12), ("box", box, 0.2), ("shell", shell, 0.15), ("shell", shell, 0.3)]


@pytest.mark.parametrize("case", range(4))
def test_shim_face_classification_matches_the_oracle(shim, case):
    name, P, alpha = clouds()[case]
    got = shim_faces(shim, P, alpha)
    assert np.all(got[:, 0] < got[:, 1]) and np.all(got[:, 1] < got[:, 2])
    assert np.array_equal(got, np.array(sorted(map(tuple, got))).reshape(-1, 3)), "faces must be in lexicographic order"
    ref, _ = oracle.alpha_faces(P.astype(np.float64), alpha)
    mine = set(map(tuple, got.tolist()))
    assert len(ref) > 100, (name, len(ref))
    assert mine == ref, (name, alpha, sorted(mine ^ ref)[:10])


def test_shim_eigen_solver_and_sign_rule(shim):
    rng = np.random.default_rng(1)
    n = 500
    B = rng.standard_normal((n, 3, 3))
    A = B @ B.transpose(0, 2, 1)
    A6 = np.ascontiguousarray(A[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]])
    d = np.ascontiguousarray(rng.standard_normal((n, 3)))
    d[0] = 0.0                                           # a tie: the largest-magnitude component is made positive
    out = np.zeros((n, 3))
    shim.shim_min_eigvec(n, A6.ctypes.data, d.ctypes.data, out.ctypes.data)
    lam, V = np.linalg.eigh(A)
    ref = V[:, :, 0]
    gap = (lam[:, 1] - lam[:, 0]) / lam.sum(1)
    ok = gap > 1e-6
    cos = np.abs((out * ref).sum(1))
    assert np.all(np.abs(np.linalg.norm(out, axis=1) - 1) < 1e-12)
    assert np.all(1 - cos[ok] < 1e-20 / gap[ok] ** 2 + 1e-12)
    s = (out * d).sum(1)
    assert np.all(s[1:] >= 0)
    assert out[0][np.argmax(np.abs(out[0]))] > 0


# ---- ABI, CLI, OBJ

@pytest.mark.parametrize("cls,cname", [(_lib.AlphaShapeArgs, "gms_alpha_shape_args"), (_lib.NormalsArgs, "gms_normals_args")])
def test_layout_matches_the_ctypes_mirror(tmp_path, cls, cname):
    body = f'    printf("size %zu\\n", sizeof({cname}));\n'
    for k in ("GMS_ALPHA_BUF_SCRATCH", "GMS_ALPHA_BUF_LISTS", "GMS_ALPHA_BUF_FACES", "GMS_ALPHA_BUF_INDEX", "GMS_ALPHA_LIST_CAP",
              "GMS_NORMALS_MAX_NN"):
        body += f'    printf("{k} %d\\n", {k});\n'
    body += "".join(f'    printf("{f[0]} %zu\\n", offsetof({cname}, {f[0]}));\n' for f in cls._fields_)
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gms_b200.h"\nint main(void) {\n' + body + "    return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).strip().split("\n"))
    assert int(out["size"]) == ctypes.sizeof(cls)
    for f in cls._fields_:
        assert int(out[f[0]]) == getattr(cls, f[0]).offset, f[0]
    assert (int(out["GMS_ALPHA_BUF_SCRATCH"]), int(out["GMS_ALPHA_BUF_LISTS"]), int(out["GMS_ALPHA_BUF_FACES"]),
            int(out["GMS_ALPHA_BUF_INDEX"])) == (_lib.ALPHA_BUF_SCRATCH, _lib.ALPHA_BUF_LISTS, _lib.ALPHA_BUF_FACES, _lib.ALPHA_BUF_INDEX)
    assert int(out["GMS_ALPHA_LIST_CAP"]) == _lib.ALPHA_LIST_CAP
    assert int(out["GMS_NORMALS_MAX_NN"]) == _lib.NORMALS_MAX_NN


def test_symbols_are_listed():
    assert {"gms_alpha_shape", "gms_normals_scratch_bytes", "gms_estimate_normals"} <= set(_lib.ABI_SYMBOLS)


def test_parser_is_the_scripts():
    from argparse import ArgumentParser
    parser = ArgumentParser(description="Testing script parameters")       # scripts/create_dummy_mesh.py, literally
    parser.add_argument("--pseudomesh_path", type=str)
    parser.add_argument("--scale", default=2, type=int)
    parser.add_argument("--alpha", default=0.003, type=float)
    mine = create_dummy_mesh.build_parser()
    for argv in ([], ["--pseudomesh_path", "a/b/triangles.pt"], ["--pseudomesh_path", "x.pt", "--scale", "3", "--alpha", "0.01"]):
        assert vars(mine.parse_args(argv)) == vars(parser.parse_args(argv))
    assert [a.dest for a in mine._actions] == [a.dest for a in parser._actions]


def test_output_name_is_the_same_for_every_alpha():
    assert create_dummy_mesh.output_path("out/pseudomesh_info/ours_30000/triangles.pt") == \
        os.path.join("out/pseudomesh_info/ours_30000", "mesh_alpha_0_003.obj")
    assert create_dummy_mesh.output_path("triangles.pt") == "mesh_alpha_0_003.obj"
    assert (create_dummy_mesh.NORMAL_RADIUS, create_dummy_mesh.NORMAL_MAX_NN) == (0.1, 30)


def test_write_obj_with_normals_round_trips(tmp_path):
    v = torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.5, 0.0], [0.25, 0.5, -2.0]])
    f = torch.tensor([[0, 1, 2], [0, 2, 3]])
    n = torch.tensor([[0.0, 0.0, 1.0], [0.0, 0.0, -1.0], [1.0, 0.0, 0.0], [0.6, 0.8, 0.0]])
    p = tmp_path / "m.obj"
    io_obj.write_obj(str(p), v, f, n)
    text = p.read_text()
    assert text.splitlines()[4] == "vn 0.000000 0.000000 1.000000"
    assert text.splitlines()[-1] == "f 1//1 3//3 4//4"
    v2, f2 = io_obj.read_obj(str(p))
    assert torch.equal(v2, v) and torch.equal(f2, f)
    with pytest.raises(ValueError, match="normals"):
        io_obj.write_obj(str(p), v, f, n[:3])


def test_write_obj_without_normals_is_unchanged(tmp_path):
    p = tmp_path / "m.obj"
    io_obj.write_obj(str(p), torch.tensor([[0.5, 0.0, -1.0], [1.0, 2.0, 3.0], [0.0, 0.0, 0.0]]), torch.tensor([[0, 1, 2]]))
    assert p.read_text() == "v 0.500000 0.000000 -1.000000\nv 1.000000 2.000000 3.000000\nv 0.000000 0.000000 0.000000\nf 1 2 3\n"


def test_empty_obj_reads_back(tmp_path):
    p = tmp_path / "e.obj"
    io_obj.write_obj(str(p), torch.zeros(0, 3), torch.zeros(0, 3, dtype=torch.int64), torch.zeros(0, 3))
    assert p.read_text() == ""
    v, f = io_obj.read_obj(str(p))
    assert v.shape == (0, 3) and f.shape == (0, 3)


def test_cpu_tensors_fail_loudly():
    from gms_b200.alpha_shape import alpha_shape, estimate_normals
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        alpha_shape(torch.zeros(4, 3), 0.1)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        estimate_normals(torch.zeros(4, 3))
