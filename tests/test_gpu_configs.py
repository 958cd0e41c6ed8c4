"""-m gpu: oracle parity on BASELINE.json's own configurations (VERDICT r1 'next round' item 1).

  * config 3 (1M mesh-Gaussians, 1920x1080): BACKWARD on every 97th tile against the oracle -- the upstream gradient is
    non-zero only on the pixels of the sampled tiles, so the GPU's full-frame backward and the oracle's strided
    composite_backward + full preprocess_backward compute the same per-Gaussian gradients;
  * config 2 (100k mesh-Gaussians, num_splats=3, 800x800): full oracle forward + backward;
  * config 4 (gs_multi_mesh, 4 meshes merged as gaussian_multi_mesh_model.py:99-119 does) at reduced P, 1080p: full oracle fwd+bwd;
  * config 5 (animated-vertex sweep, scripts/render_time_animated.py:34-40,68-87) at 3 values of t: forward vs oracle.
Every test prints the threshold-ambiguous pixel count and the measured maxima."""
import numpy as np
import pytest
import torch

import bench
import diff_gaussian_rasterization as dgr
from gms_b200 import rasterizer, scenes
from gms_b200.model import MeshGaussianModel, MultiMeshGaussianModel
from gpu_helpers import assert_forward_parity, assert_grad_parity, gpu_settings, run_gpu, run_oracle
from helpers import settings_from_camera
from oracle import raster

pytestmark = pytest.mark.gpu


def _model_inputs(model):
    with torch.no_grad():
        xyz, sc, rot = model.expand_fused(activated=True)
        return dict(means3D=xyz.cpu(), scales=sc.cpu(), rotations=rot.cpu(), opacities=model.get_opacity.cpu(),
                    shs=model.get_features.cpu().contiguous())


def test_config3_sampled_tile_backward_matches_oracle_at_full_size():
    params, cams, dims = bench.build_scene("gs_mesh_1M_1080p")
    F, K, W, H = dims
    model = MeshGaussianModel.from_params(params, "cuda", packed_features=True)
    cam = cams[2]
    S = settings_from_camera(cam, bg=(1, 1, 1))
    inputs = _model_inputs(model)
    gx, stride = (W + 15) // 16, 97
    rs = np.random.RandomState(7)
    dC = np.zeros((3, H, W), np.float32)
    T = gx * ((H + 15) // 16)
    for tile in range(0, T, stride):
        x0, y0 = (tile % gx) * 16, (tile // gx) * 16
        dC[:, y0:y0 + 16, x0:x0 + 16] = rs.randn(3, min(16, H - y0), min(16, W - x0)).astype(np.float32) / 256.0
    color, radii, invd, state, g = run_gpu(S, inputs, dC)
    st = raster.preprocess(S, inputs["means3D"], inputs["opacities"], shs=inputs["shs"], scales=inputs["scales"], rotations=inputs["rotations"])
    np.testing.assert_array_equal(st.radii, radii)
    raster.bin_tiles(st)
    np.testing.assert_array_equal(st.point_list, state["point_list"].astype(np.uint32))
    raster.set_tile_stride(stride)
    try:
        raster.composite(st)
        gc = raster.composite_backward(st, dC, None)
    finally:
        raster.set_tile_stride(1)
    go = raster.preprocess_backward(st, gc)
    go["_composite"] = gc
    go["_upstream"] = (dC, None)       # zero outside the sampled tiles, where n_contrib is 0 as well
    # forward on the sampled tiles
    worst, amb = 0.0, 0
    for tile in range(0, T, stride):
        x0, y0 = (tile % gx) * 16, (tile // gx) * 16
        sl = (slice(None), slice(y0, min(y0 + 16, H)), slice(x0, min(x0 + 16, W)))
        ok = st.ambiguous[sl[1:]] == 0
        amb += int((~ok).sum())
        worst = max(worst, float(np.abs(color[sl] - st.color[sl])[:, ok].max()) if ok.any() else 0.0)
    print(f"[config 3] P={F * K} N={st.N} sampled tiles={len(range(0, T, stride))} ambiguous px={amb} max|image-oracle|={worst:.2e}")
    assert worst <= 1e-5
    touched = np.abs(go["dL_dsh"]).reshape(F * K, -1).max(axis=1) > 0
    assert touched.sum() > 1000
    assert_grad_parity(g, go, st=st)


def test_config2_full_frame_forward_and_backward_match_oracle():
    params, cams, dims = bench.build_scene("gs_mesh_100k_800")
    model = MeshGaussianModel.from_params(params, "cuda")
    S = settings_from_camera(cams[3], bg=(1, 1, 1))
    inputs = _model_inputs(model)
    rs = np.random.RandomState(2)
    dC = (rs.randn(3, 800, 800) / (800 * 800)).astype(np.float32)
    color, radii, invd, state, g = run_gpu(S, inputs, dC)
    st, go = run_oracle(S, inputs, dC)
    print(f"[config 2] P={inputs['means3D'].shape[0]} N={st.N}")
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(g, go, st=st)


def test_config4_multi_mesh_reduced_matches_oracle():
    plist = []
    for k, c in enumerate([(-0.75, -0.75, 0.0), (0.75, -0.75, 0.0), (-0.75, 0.75, 0.0), (0.75, 0.75, 0.0)]):
        v, f = scenes.object_mesh(6000)
        plist.append(scenes.init_mesh_gaussians(v * 0.55 + np.float32(c), f, 5, seed=20 + k, trained_like=True))
    model = MultiMeshGaussianModel.from_mesh_params(plist, "cuda")
    cam = scenes.ring_cameras(4, 3.6, 1920, 1080, elevation_deg=25.0)[1]
    S = settings_from_camera(cam, bg=(1, 1, 1))
    inputs = _model_inputs(model)
    rs = np.random.RandomState(3)
    dC = (rs.randn(3, 1080, 1920) / (1080 * 1920)).astype(np.float32)
    color, radii, invd, state, g = run_gpu(S, inputs, dC)
    st, go = run_oracle(S, inputs, dC)
    print(f"[config 4, reduced] meshes=4 P={inputs['means3D'].shape[0]} N={st.N}")
    assert_forward_parity(st, color, radii, invd, state)
    assert_grad_parity(g, go, st=st)


@pytest.mark.parametrize("t", [0.0, 9.7, 10 * np.pi])
def test_config5_animated_frames_match_oracle(t):
    params, cams, dims = bench.build_scene("gs_mesh_100k_800")
    model = MeshGaussianModel.from_params(params, "cuda")
    v0 = model.vertices.detach().clone()
    with torch.no_grad():
        model.vertices.data.copy_(scenes.transform_hotdog_fly(v0, float(t)))
    cam = scenes.ring_cameras(3, 3.4, 1920, 1080, elevation_deg=15.0)[0]
    S = settings_from_camera(cam, bg=(1, 1, 1))
    inputs = _model_inputs(model)
    color, radii, invd, state, _ = run_gpu(S, inputs)
    st, _ = run_oracle(S, inputs)
    print(f"[config 5] t={t:.2f} N={st.N}")
    assert_forward_parity(st, color, radii, invd, state)
