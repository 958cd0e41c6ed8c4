"""-m gpu: initialising gs / gs_flat models from a point cloud.  gms_knn_dist2 against the float32 oracle (tests/knn_oracle.py)
bit for bit on the clouds where a pruned search could go wrong; its argument checks; the simple_knn drop-in;
FreeGaussianModel.from_point_cloud against the reference's create_from_pcd (tests/golden/pcd_init.npz); and a short gs_flat
training run from the reference's random NeRF-synthetic cloud."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import knn_oracle as K
from gms_b200 import _lib, knn, scenes
from gms_b200.model import FreeGaussianModel
from gms_b200.render import NativeFreeRenderer
from gms_b200.trainer import FreeOptimizationParams, FreeTrainer
from helpers import random_gaussians

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = _lib.KNN_BOX


def _native(pts: np.ndarray) -> np.ndarray:
    out = knn.mean_dist2(torch.from_numpy(np.ascontiguousarray(pts, np.float32)).cuda())
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _assert_bits(got: np.ndarray, ref: np.ndarray, what: str):
    assert got.dtype == ref.dtype == np.float32 and got.shape == ref.shape, what
    bad = np.flatnonzero(got.view(np.uint32) != ref.view(np.uint32))
    assert bad.size == 0, f"{what}: {bad.size} of {got.size} rows differ, first {bad[:5]}: {got[bad[:5]]} vs {ref[bad[:5]]}"


def _straddling(seed=0) -> np.ndarray:
    """A cloud whose box is [-1,1]^3 (its corners are in it), so the top Morton split plane is x = 0: a 40 x 40 grid of pairs
    at x = +-1e-4 (spacing 0.05 in y, z) whose nearest neighbours lie across the plane, many boxes away in sort order; plus
    a 16^3 lattice with every coordinate on a Morton cell boundary (k/8 - 1)."""
    corners = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64)
    g = np.linspace(-0.975, 0.975, 40)
    yy, zz = np.meshgrid(g, g, indexing="ij")
    plane = np.stack([np.zeros(yy.size), yy.ravel(), zz.ravel()], 1)
    pairs = np.concatenate([plane + [1e-4, 0, 0], plane - [1e-4, 0, 0]])
    k = np.arange(16) / 8.0 - 1
    lat = np.stack(np.meshgrid(k, k, k, indexing="ij"), -1).reshape(-1, 3) + [0.0, 0.0, 0.03]
    pts = np.concatenate([corners, pairs, lat]).astype(np.float32)
    return pts[np.random.default_rng(seed).permutation(pts.shape[0])]


def _collinear(seed=0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    on_x = np.zeros((6000, 3), np.float32)
    on_x[:, 0] = rng.uniform(-3, 3, 6000)
    return on_x


def test_reference_random_cloud_100k():
    pts = scenes.random_point_cloud(100_000, 0)[0]
    _assert_bits(_native(pts), K.dist2(pts), "random 100k")


def test_clustered_1m_and_deterministic():
    pts = K.surface_points(1_000_000, seed=1)
    t = torch.from_numpy(pts).cuda()
    a, b = knn.mean_dist2(t), knn.mean_dist2(t)
    torch.cuda.synchronize()
    a, b = a.cpu().numpy(), b.cpu().numpy()
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "two calls differ"
    _assert_bits(a, K.dist2(pts), "clustered 1M")


def test_every_point_duplicated():
    rng = np.random.default_rng(2)
    half = rng.uniform(-1, 1, (30_000, 3)).astype(np.float32)
    pts = np.concatenate([half, half])[rng.permutation(60_000)]
    got = _native(pts)
    _assert_bits(got, K.dist2(pts), "duplicated")
    assert (got > 0).all()       # b0 = 0 (the twin), b1, b2 > 0


def test_all_points_identical_clamps_the_scale():
    pts = np.tile(np.array([[0.25, -3.0, 7.0]], np.float32), (5000, 1))
    got = _native(pts)
    assert (got.view(np.uint32) == 0).all()
    m = FreeGaussianModel.from_point_cloud(pts, np.full(pts.shape, 0.5), "gs")
    ref = torch.log(torch.sqrt(torch.clamp_min(torch.zeros(1, device="cuda"), 0.0000001)))
    assert torch.equal(m._scaling.detach(), ref.expand(5000, 3))


@pytest.mark.parametrize("name", ["collinear", "straddling", "offset_1e4"])
def test_degenerate_and_adversarial_layouts(name):
    rng = np.random.default_rng(3)
    if name == "collinear":
        pts = _collinear()
        pts = np.concatenate([pts, pts[:2000][:, [1, 0, 2]] + np.float32(5)])    # a second line, along y
    elif name == "straddling":
        pts = _straddling()
    else:
        pts = (rng.uniform(0, 8, (20_000, 3)) + 1e4).astype(np.float32)
    _assert_bits(_native(pts), K.brute(pts), name)


@pytest.mark.parametrize("P", [4, 5, B - 1, B, B + 1, 2 * B + 3, 1000])
def test_small_and_partial_box_sizes(P):
    rng = np.random.default_rng(P)
    pts = rng.normal(size=(P, 3)).astype(np.float32)
    if P >= 10:
        pts[P // 2] = pts[1]                               # a duplicate pair
    _assert_bits(_native(pts), K.brute(pts), f"P={P}")


def test_arguments():
    assert knn.mean_dist2(torch.zeros(0, 3, device="cuda")).shape == (0,)
    for P in (1, 2, 3):
        with pytest.raises(ValueError, match="three neighbours"):
            knn.mean_dist2(torch.zeros(P, 3, device="cuda"))
    with pytest.raises(RuntimeError, match="CUDA"):
        knn.mean_dist2(torch.zeros(8, 3))
    for bad in (float("nan"), float("inf")):
        x = torch.zeros(8, 3, device="cuda")
        x[5, 1] = bad
        with pytest.raises(ValueError, match="finite"):
            knn.mean_dist2(x)
    with pytest.raises(ValueError):
        knn.mean_dist2(torch.zeros(8, 2, device="cuda"))
    # the C entry point's own checks: P in 1..3, a null pointer, too little scratch; P = 0 is a no-op
    L = _lib.lib()
    pts = torch.rand(100, 3, device="cuda")
    out = torch.empty(100, device="cuda")
    need = int(L.gms_knn_scratch_bytes(100))
    scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def call(P, points, dist2, nbytes):
        a = _lib.KnnArgs()
        a.P, a.points, a.dist2, a.scratch, a.scratch_bytes = P, points, dist2, scratch.data_ptr(), nbytes
        return L.gms_knn_dist2(C.byref(a), st)

    assert call(0, None, None, 0) == _lib.GMS_OK
    for P in (1, 2, 3, -1):
        assert call(P, pts.data_ptr(), out.data_ptr(), need) == _lib.GMS_E_ARG
    assert call(100, None, out.data_ptr(), need) == _lib.GMS_E_ARG
    assert call(100, pts.data_ptr(), None, need) == _lib.GMS_E_ARG
    assert call(100, pts.data_ptr(), out.data_ptr(), need - 1) == _lib.GMS_E_ARG
    assert call(100, pts.data_ptr(), out.data_ptr(), need) == _lib.GMS_OK
    torch.cuda.synchronize()
    _assert_bits(out.cpu().numpy(), K.brute(pts.cpu().numpy()), "direct call")


def test_simple_knn_drop_in():
    from simple_knn._C import distCUDA2
    pts = torch.from_numpy(K.surface_points(50_000, seed=4)).cuda()
    assert torch.equal(distCUDA2(pts), knn.mean_dist2(pts))


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "pcd_init.npz")))


def _ulps(a: torch.Tensor, b: np.ndarray) -> int:
    x = a.detach().cpu().numpy().astype(np.float32).view(np.int32).astype(np.int64)
    y = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    return int(np.abs(x - y).max())


@pytest.mark.parametrize("kind", ["gs", "gs_flat"])
def test_from_point_cloud_matches_create_from_pcd(golden, kind):
    pts, colors = golden["pcd_points"], golden["pcd_colors"]
    _assert_bits(_native(pts.astype(np.float32)), golden["pcd_dist2"], "fixture cloud")
    m = FreeGaussianModel.from_point_cloud(pts, colors, kind)
    g = lambda n: golden[f"{kind}{n}"]
    assert m.kind == kind and m.active_sh_degree == int(g("_active_sh_degree")) == 0 and m.max_sh_degree == 3
    assert np.array_equal(m._xyz.detach().cpu().numpy(), g("_xyz"))
    assert np.array_equal(m._features.detach().cpu().numpy(), np.concatenate([g("_features_dc"), g("_features_rest")], 1))
    assert np.array_equal(m._rotation.detach().cpu().numpy(), g("_rotation"))
    assert m._scaling.shape == g("_scaling").shape and _ulps(m._scaling, g("_scaling")) <= 1
    assert _ulps(m._opacity, g("_opacity")) <= 1


def test_training_run_from_the_random_cloud(tmp_path):
    """gs_flat from the reference's random 100k-style cloud (10k points), white background, 600 iterations at 256x256
    against targets rendered from another model, densifying from 200: no overflowed frame, the loss falls, and the
    checkpoint reloads."""
    W = H = 256
    cams = [c.to("cuda") for c in scenes.ring_cameras(8, 2.5, W, H)]
    for i, c in enumerate(cams):
        c.uid = i
    white = torch.ones(3, device="cuda")
    g = random_gaussians(4000, seed=21, extent=0.8, flat_frac=0.0)
    target = FreeGaussianModel(g["means3D"], torch.log(g["scales"][:, 1:]).contiguous(), g["rotations"], g["shs"],
                               torch.logit(g["opacities"]), "gs_flat", "cuda", 0)
    rt = NativeFreeRenderer(target, W, H)
    gts = [rt.render(c, white)[0].clone() for c in cams]
    pts, colors, _ = scenes.random_point_cloud(10_000, 0)
    model = FreeGaussianModel.from_point_cloud(pts, colors, "gs_flat")
    o = FreeOptimizationParams(iterations=600, densify_from_iter=200, densification_interval=100)
    tr = FreeTrainer(model, white, scenes.camera_extent(cams), o)
    losses = torch.stack([tr.step(cams[it % len(cams)], gts[it % len(cams)]).clone() for it in range(1, 601)]).cpu()
    assert tr.frame.overflows == 0
    assert len(tr.densifications) == 4 and model.P != 10_000
    first, last = float(losses[:50].mean()), float(losses[-50:].mean())
    print(f"[pcd training] P 10000 -> {model.P}, loss {first:.4f} -> {last:.4f}")
    assert last < 0.9 * first
    ply = str(tmp_path / "point_cloud.ply")
    model.save(ply)
    back = FreeGaussianModel.from_checkpoint(ply, "gs_flat", "cuda")
    assert torch.equal(back._xyz, model._xyz.detach()) and torch.equal(back._scaling, model._scaling.detach())
    assert torch.equal(back._features, model._features.detach()) and torch.equal(back._opacity, model._opacity.detach())
