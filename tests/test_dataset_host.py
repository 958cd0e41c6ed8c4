"""Host half of the dataset loader (gms_b200/dataset.py) against tests/golden/dataset.npz, written by the reference's own
readers (tests/golden/make_dataset_golden.py), and the resample tables against tests/resize_oracle.py.  No GPU."""
import hashlib
import os
import shutil

import numpy as np
import pytest
import torch

import dataset_cases
import resize_oracle
from gms_b200 import dataset

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "dataset.npz"))


@pytest.fixture(scope="module")
def datasets(tmp_path_factory):
    return dataset_cases.write_all(str(tmp_path_factory.mktemp("datasets")))


def _tree_digest(root):
    h = hashlib.sha256()
    for d, _, files in sorted(os.walk(root)):
        for f in sorted(files):
            p = os.path.join(d, f)
            h.update(os.path.relpath(p, root).encode())
            h.update(open(p, "rb").read())
    return h.hexdigest()


def _ulp_close(a, b, ulps=1):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    tol = ulps * np.spacing(np.maximum(np.abs(a), np.abs(b)))
    return bool(np.all(np.abs(a.astype(np.float64) - b.astype(np.float64)) <= np.maximum(tol, 1e-30)))


@pytest.mark.parametrize("case", sorted(dataset_cases.CASES))
def test_read_scene_matches_reference(case, datasets):
    ds, kw = dataset_cases.CASES[case]
    before = _tree_digest(datasets[ds])
    sc = dataset.read_scene(datasets[ds], **kw)
    assert _tree_digest(datasets[ds]) == before, "the loader wrote into the source directory"
    g = {k[len(case) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(case + "/")}
    assert sc.cameras_extent == pytest.approx(float(g["extent"]), rel=1e-6)
    assert sc.view_order(40) == g["order"].tolist()
    for split, cams, views in (("train", sc.train_cameras, sc.train_views), ("test", sc.test_cameras, sc.test_views)):
        assert [v.name for v in views] == g[f"{split}/names"].tolist()
        assert len(cams) == len(g[f"{split}/names"])
        for i, (c, v) in enumerate(zip(cams, views)):
            assert c.uid == i
            assert np.array_equal(v.R, g[f"{split}/R"][i]) and np.array_equal(v.T, g[f"{split}/T"][i])
            assert (c.FoVx, c.FoVy) == tuple(g[f"{split}/fov"][i])
            assert (c.image_width, c.image_height) == tuple(g[f"{split}/size"][i])
            assert tuple(g[f"{split}/image{i}"].shape) == (c.image_height, c.image_width, 3)
            for n in ("world_view_transform", "full_proj_transform", "camera_center"):
                assert _ulp_close(getattr(c, n).numpy(), g[f"{split}/{n}"][i]), (split, i, n)
    if kw["gs_type"] == "gs_mesh":
        m = sc.mesh
        for n in ("vertices", "faces", "_alpha", "_scale", "_features_dc", "_features_rest", "_opacity"):
            assert np.array_equal(getattr(m, n).numpy(), g[f"mesh{n}"]), n
    else:
        for k, a in zip(("points", "colors", "normals"), sc.point_cloud):
            assert np.array_equal(a[:len(g[f"pcd_{k}"])], g[f"pcd_{k}"]), k
            assert str(g[f"pcd_{k}_meta"]) == f"{a.dtype.str} {a.shape[0]}x{a.shape[1]}"
            assert hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest() == str(g[f"pcd_{k}_sha256"])


def test_view_order_is_repeatable(datasets):
    sc = dataset.read_scene(datasets["blender_a"], "gs")
    assert sc.view_order(25) == sc.view_order(25)
    assert sorted(sc.view_order(5)) == list(range(5))       # one pass over the five views before the stack refills


def test_camera_resolution_rules():
    assert dataset.camera_resolution(25, 17, 2) == (12, 8)          # round halves to even
    assert dataset.camera_resolution(27, 17, 2) == (14, 8)
    assert dataset.camera_resolution(1601, 900, -1)[0] == 1599
    assert dataset.camera_resolution(1617, 900, -1)[0] == 1599
    assert dataset.camera_resolution(4946, 3286, -1) == (1600, 1063)
    assert dataset.camera_resolution(1600, 900, -1) == (1600, 900)
    assert dataset.camera_resolution(50, 36, 40) == (40, 28)
    assert dataset.camera_resolution(30, 20, 31) == (31, 20)
    # the 1599 quirk: int(w / (w / 1600)) for every width the automatic downscale touches
    n1599 = sum(int(w / (w / 1600)) == 1599 for w in range(1601, 8001))
    assert n1599 == sum(dataset.camera_resolution(w, 1000, -1)[0] == 1599 for w in range(1601, 8001)) == 464
    with pytest.raises(ValueError):
        dataset.camera_resolution(1, 1, 2)
    with pytest.raises(ValueError):
        dataset.camera_resolution(3000, 1, -1)


@pytest.mark.parametrize("n_in,n_out", [(37, 18), (23, 11), (800, 400), (160, 50), (90, 28), (67, 33), (64, 80), (48, 60),
                                        (333, 160), (211, 101), (1601, 1599), (4946, 1600), (3286, 1063), (5, 1), (1, 7),
                                        (9000, 1600), (3, 3)])
def test_resize_tables_match_oracle(n_in, n_out):
    b, k = dataset.resize_coeffs(n_in, n_out)
    ob, ok, ksize = resize_oracle.coeffs(n_in, n_out)
    assert k.shape == (n_out, ksize)
    assert b.tolist() == [list(x) for x in ob]
    assert k.tolist() == ok


def test_resize_oracle_matches_pillow():
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(11)
    pairs = [((37, 23), (18, 11)), ((101, 67), (101, 33)), ((64, 48), (80, 60)), ((160, 90), (50, 28)), ((40, 30), (41, 30))]
    for _ in range(20):
        W, H = rng.integers(1, 120, 2)
        w, h = rng.integers(1, 160, 2)
        pairs.append(((int(W), int(H)), (int(w), int(h))))
    for (W, H), (w, h) in pairs:
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        ref = np.asarray(Image.fromarray(img, "RGB").resize((w, h)))
        assert np.array_equal(resize_oracle.resize(img, w, h), ref), ((W, H), (w, h))


def test_composite_oracle_is_the_truncated_sequence():
    v, a = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    rgba = np.stack([v, v, v, a], -1).astype(np.uint8)
    for white in (False, True):
        n = rgba / 255.0
        seq = n[..., :3] * n[..., 3:4] + (1.0 if white else 0.0) * (1 - n[..., 3:4])
        assert np.array_equal(resize_oracle.composite(rgba, white), np.trunc(seq * 255.0).astype(np.uint8))


def test_unsupported_camera_model_and_mode(datasets, tmp_path):
    with pytest.raises(ValueError, match="OPENCV"):
        dataset.read_scene(datasets["colmap_opencv"], "gs")
    path = os.path.join(datasets["colmap_rgba"], "images")
    first = sorted(os.listdir(path))
    with pytest.raises(ValueError, match="RGBA"):
        for f in first:
            dataset.decode_image(os.path.join(path, f), "RGB")
    with pytest.raises(ValueError, match="gs_mesh"):
        dataset.read_scene(datasets["colmap_bin"], "gs_mesh")
    with pytest.raises(ValueError):
        dataset.read_scene(str(tmp_path), "gs")


def test_decode_without_pillow_matches(datasets, monkeypatch):
    """The PNG fallback expands to RGBA as convert("RGBA") does."""
    Image = pytest.importorskip("PIL.Image")
    p = os.path.join(datasets["blender_a"], "train", "r_0.png")
    with_pil = dataset.decode_image(p, "RGBA")
    import builtins
    real_import = builtins.__import__

    def no_pil(name, *a, **k):
        if name == "PIL" or name.startswith("PIL."):
            raise ImportError(name)
        return real_import(name, *a, **k)

    monkeypatch.setattr(builtins, "__import__", no_pil)
    assert np.array_equal(dataset.decode_image(p, "RGBA"), with_pil)
    rgb = os.path.join(datasets["colmap_bin"], "images", sorted(os.listdir(os.path.join(datasets["colmap_bin"], "images")))[0])
    grey = np.arange(12, dtype=np.uint8).reshape(3, 4, 1)
    gp = os.path.join(str(os.path.dirname(p)), "..", "grey.png")
    dataset_cases.write_png(gp, grey)
    exp = np.concatenate([np.repeat(grey, 3, 2), np.full((3, 4, 1), 255, np.uint8)], 2)
    assert np.array_equal(dataset.decode_image(gp, "RGBA"), exp)
    os.remove(gp)
    assert dataset.decode_image(rgb, "RGB").shape[2] == 3
