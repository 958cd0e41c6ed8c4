"""point_cloud.ply IO without plyfile: layout of GaussianModel._save_ply / _load_ply (scene/gaussian_model.py:177-262)."""
import os

import numpy as np
import pytest
import torch

from gms_b200 import io_ply, scenes


def _random_model(P=37, M=16, S=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    return r(P, 3), r(P, 1, 3), r(P, M - 1, 3), r(P, 1), r(P, S), r(P, 4)


def test_round_trip_and_reference_property_order(tmp_path):
    xyz, fdc, frest, op, sc, rot = _random_model()
    p = str(tmp_path / "point_cloud.ply")
    io_ply.save_gaussian_ply(p, xyz, fdc, frest, op, sc, rot)
    data, names = io_ply.read_ply_vertices(p)
    expect = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(45)] + \
             ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    assert names == expect                                    # construct_list_of_attributes, scene/gaussian_model.py:170-183
    # channel-major SH: f_rest_k holds coefficient (k % 15) + 1 of channel k // 15   (transpose(1,2).flatten, :191-192)
    np.testing.assert_array_equal(np.asarray(data["f_rest_17"]), frest[:, 2, 1].numpy())
    np.testing.assert_array_equal(np.asarray(data["f_dc_1"]), fdc[:, 0, 1].numpy())
    g = io_ply.load_gaussian_ply(p)
    for k, v in dict(_xyz=xyz, _features_dc=fdc, _features_rest=frest, _opacity=op, _scaling=sc, _rotation=rot).items():
        assert g[k].shape == v.shape and torch.equal(g[k], v), k


def test_ascii_ply_and_flat_two_scale_models(tmp_path):
    xyz, fdc, frest, op, sc, rot = _random_model(P=5, S=2)
    p = str(tmp_path / "a.ply")
    cols = torch.cat([xyz, torch.zeros(5, 3), fdc.transpose(1, 2).reshape(5, -1), frest.transpose(1, 2).reshape(5, -1), op, sc, rot], 1)
    names = ["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(3)] + [f"f_rest_{i}" for i in range(45)] + ["opacity", "scale_0", "scale_1"] + [f"rot_{i}" for i in range(4)]
    with open(p, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex 5\n" + "".join(f"property float {n}\n" for n in names) + "end_header\n")
        for row in cols.numpy():
            f.write(" ".join(repr(float(v)) for v in row) + "\n")
    g = io_ply.load_gaussian_ply(p)
    assert g["_scaling"].shape == (5, 2)
    np.testing.assert_allclose(g["_features_rest"].numpy(), frest.numpy(), rtol=1e-6)
    np.testing.assert_allclose(g["_xyz"].numpy(), xyz.numpy(), rtol=1e-6)


def test_mesh_model_params_round_trip(tmp_path):
    """model_params.pt next to the PLY (gaussian_mesh_model.py:189-225): what load_mesh_model returns re-creates the model."""
    p = scenes.init_mesh_gaussians(*scenes.icosphere(1), K=2, seed=3)
    ply = str(tmp_path / "point_cloud" / "iteration_7" / "point_cloud.ply")
    os.makedirs(os.path.dirname(ply))
    io_ply.save_gaussian_ply(ply, torch.zeros(p.P, 3), p._features_dc, p._features_rest, p._opacity, torch.zeros(p.P, 3), torch.zeros(p.P, 4))
    torch.save({"_alpha": p._alpha, "_scale": p._scale, "vertices": p.vertices, "faces": p.faces, "triangles": p.vertices[p.faces]},
               ply.replace("point_cloud.ply", "model_params.pt"))
    q = io_ply.load_mesh_model(ply)
    for k in ("vertices", "faces", "_alpha", "_scale", "_features_dc", "_features_rest", "_opacity"):
        assert torch.equal(getattr(p, k), getattr(q, k)), k


def test_reads_a_checkpoint_written_by_the_reference(golden_dir):
    """tests/golden/ply/ was written by the reference's own GaussianMeshModel.save_ply (tests/golden/make_ply_golden.py):
    property order, channel-major SH layout and the model_params.pt keys are the reference's, not this repo's writer's."""
    ply = os.path.join(golden_dir, "ply", "point_cloud.ply")
    want = np.load(os.path.join(golden_dir, "ply", "expected.npz"))
    g = io_ply.load_gaussian_ply(ply)
    for k in ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"):
        np.testing.assert_array_equal(g[k].numpy(), want[k])
    p = io_ply.load_mesh_model(ply)
    for k in ("vertices", "faces", "_alpha", "_scale", "_opacity", "_features_dc", "_features_rest"):
        np.testing.assert_array_equal(getattr(p, k).numpy(), want[k])
    assert p.faces.dtype == torch.int64


def test_two_column_scaling_gets_the_s0_column_like_the_reference(tmp_path):
    xyz, fdc, frest, op, sc, rot = _random_model(P=11, S=2)
    p = str(tmp_path / "point_cloud.ply")
    io_ply.save_gaussian_ply(p, xyz, fdc, frest, op, sc, rot)
    data, names = io_ply.read_ply_vertices(p)
    assert [n for n in names if n.startswith("scale_")] == ["scale_0", "scale_1", "scale_2"]       # scene/gaussian_model.py:179-180
    np.testing.assert_allclose(np.asarray(data["scale_0"]), np.log(np.float32(1e-8)), rtol=1e-6)
    np.testing.assert_array_equal(np.asarray(data["scale_2"]), sc[:, 1].numpy())


@pytest.mark.parametrize("M", [1, 4, 9])
def test_round_trip_below_sixteen_coefficients(tmp_path, M):
    """--sh_degree 0, 1, 2: 3 * (M - 1) f_rest properties (none at degree 0), channel-major, and [P, M - 1, 3] on load."""
    xyz, fdc, frest, op, sc, rot = _random_model(P=13, M=M, seed=M)
    p = str(tmp_path / "point_cloud.ply")
    io_ply.save_gaussian_ply(p, xyz, fdc, frest, op, sc, rot)
    data, names = io_ply.read_ply_vertices(p)
    n_rest = 3 * (M - 1)
    assert names == ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(n_rest)] + \
        ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    for k in range(n_rest):        # f_rest_k holds coefficient (k % (M - 1)) + 1 of channel k // (M - 1)
        np.testing.assert_array_equal(np.asarray(data[f"f_rest_{k}"]), frest[:, k % (M - 1), k // (M - 1)].numpy())
    g = io_ply.load_gaussian_ply(p)
    assert g["_features_rest"].shape == (13, M - 1, 3)
    for k, v in dict(_xyz=xyz, _features_dc=fdc, _features_rest=frest, _opacity=op, _scaling=sc, _rotation=rot).items():
        assert g[k].shape == v.shape and torch.equal(g[k], v), k
    back = torch.cat((g["_features_dc"], g["_features_rest"]), 1)
    assert back.shape == (13, M, 3) and torch.equal(back, torch.cat((fdc, frest), 1))


def _write_ply(path, names, rows):
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % rows.shape[0]).encode())
        for n in names:
            f.write(f"property float {n}\n".encode())
        f.write(b"end_header\n")
        np.ascontiguousarray(rows, "<f4").tofile(f)


@pytest.mark.parametrize("n_rest,n_dc", [(3, 3), (6, 3), (12, 3), (44, 3), (48, 3), (9, 2), (0, 0)])
def test_refuses_sh_property_counts_of_no_degree(tmp_path, n_rest, n_dc):
    """f_rest counts other than 0, 9, 24 and 45 (or f_dc counts other than 3) name no SH degree 0..3: refused by name."""
    names = ["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(n_dc)] + [f"f_rest_{i}" for i in range(n_rest)] + \
        ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    p = str(tmp_path / "bad.ply")
    _write_ply(p, names, np.random.RandomState(0).randn(4, len(names)))
    with pytest.raises(ValueError, match=rf"{n_dc} f_dc_\* and {n_rest} f_rest_\* properties"):
        io_ply.load_gaussian_ply(p)


@pytest.mark.parametrize("M", [1, 4, 9, 16])
def test_free_model_checkpoint_keeps_its_coefficient_count(tmp_path, M):
    """FreeGaussianModel.save -> from_checkpoint (on the CPU): features [P, M, 3] and max_sh_degree from M."""
    from gms_b200.model import FreeGaussianModel
    xyz, fdc, frest, op, sc, rot = _random_model(P=9, M=M, S=2, seed=20 + M)
    m = FreeGaussianModel(xyz, sc, rot, torch.cat((fdc, frest), 1), op, "gs_flat", "cpu", active_sh_degree=3)
    assert m.max_sh_degree == m.active_sh_degree == int(round(M ** 0.5)) - 1
    p = str(tmp_path / "point_cloud.ply")
    m.save(p)
    back = FreeGaussianModel.from_checkpoint(p, "gs_flat", "cpu")
    assert back._features.shape == (9, M, 3) and torch.equal(back._features, m._features.detach())
    assert back.max_sh_degree == m.max_sh_degree
