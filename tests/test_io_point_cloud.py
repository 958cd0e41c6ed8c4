"""CPU-only: the point clouds a gs / gs_flat run starts from.  scenes.random_point_cloud is the cloud readNerfSyntheticInfo
trains from, after its storePly -> fetchPly round trip (tests/golden/pcd_init.npz, written by the reference's own code);
io_ply.save_point_cloud / load_point_cloud are storePly / fetchPly; ASCII and binary PLY read the same."""
import hashlib
import os

import numpy as np
import pytest

from gms_b200 import io_ply, scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "pcd_init.npz")))


def _check(arrays, golden):
    for n, a in zip(("points", "colors", "normals"), arrays):
        rows = golden[f"nerf_{n}"]
        assert f"{a.dtype.str} {a.shape[0]}x{a.shape[1]}" == str(golden[f"nerf_{n}_meta"]), n
        assert a.dtype == rows.dtype and np.array_equal(a[:rows.shape[0]], rows), n
        assert hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest() == str(golden[f"nerf_{n}_sha256"]), n


def test_random_point_cloud_matches_the_reference(golden):
    pts, colors, normals = scenes.random_point_cloud(100_000, 0)
    _check((pts, colors, normals), golden)
    assert pts.dtype == np.float32 and pts.min() >= -1.3 and pts.max() <= 1.3
    assert (colors == 127 / 255).all() and (normals == 0).all()      # the byte truncation of storePly


def test_save_then_load_round_trips_to_the_reference(golden, tmp_path):
    rng = np.random.RandomState(0)
    xyz = rng.random_sample((100_000, 3)) * 2.6 - 1.3
    shs = rng.random_sample((100_000, 3)) / 255.0
    path = str(tmp_path / "points3d.ply")
    io_ply.save_point_cloud(path, xyz, (shs * scenes.SH_C0 + 0.5) * 255)
    _check(io_ply.load_point_cloud(path), golden)
    with open(path, "rb") as f:
        head = f.read(400).split(b"end_header\n")[0].decode()
    assert "format binary_little_endian 1.0" in head and "element vertex 100000" in head
    assert head.index("property float nz") < head.index("property uchar red") < head.index("property uchar blue")


def test_colour_bytes_truncate(tmp_path):
    path = str(tmp_path / "c.ply")
    io_ply.save_point_cloud(path, np.zeros((3, 3)), np.array([[0.9, 127.99, 254.6], [1.0, 2.5, 3.999], [255.0, 0.0, 100.5]]))
    _, colors, _ = io_ply.load_point_cloud(path)
    assert np.array_equal(np.round(colors * 255), [[0, 127, 254], [1, 2, 3], [255, 0, 100]])


def test_ascii_and_binary_point_clouds_read_the_same(tmp_path):
    rng = np.random.default_rng(3)
    xyz = rng.uniform(-2, 2, (50, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (50, 3))
    b = str(tmp_path / "bin.ply")
    io_ply.save_point_cloud(b, xyz, rgb)
    a = str(tmp_path / "ascii.ply")
    with open(a, "w") as f:
        f.write("ply\nformat ascii 1.0\ncomment written by hand\nelement vertex 50\n")
        for n in ("x", "y", "z", "nx", "ny", "nz"):
            f.write(f"property float {n}\n")
        for n in ("red", "green", "blue"):
            f.write(f"property uchar {n}\n")
        f.write("end_header\n")
        for p, c in zip(xyz, rgb):
            f.write(" ".join(f"{v:.9g}" for v in p) + " 0 0 0 " + " ".join(str(int(v)) for v in c) + "\n")
    for x, y in zip(io_ply.load_point_cloud(a), io_ply.load_point_cloud(b)):
        assert x.dtype == y.dtype and np.array_equal(x, y)
    assert np.array_equal(io_ply.load_point_cloud(b)[0], xyz)
