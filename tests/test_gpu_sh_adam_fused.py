"""-m gpu: the SH Adam step applied inside the preprocess backward of a single-GPU training frame (gms_train_frame with
gms_sh_adam) is bit for bit the step gms_adam_sh_factored takes from the same frame's colour gradients."""
import ctypes as C

import pytest
import torch

from gms_b200 import _lib, scenes
from gms_b200.model import MeshGaussianModel
from gms_b200.optim import FlatAdam, mesh_model_groups
from gms_b200.trainer import NativeFrame, render_frame

pytestmark = pytest.mark.gpu

W, H = 352, 256


def _scene():
    verts, faces = scenes.icosphere(3)
    # 1277 faces x 3 = 3831 Gaussians: the last warp of 32 rows is partly out of bounds
    p = scenes.init_mesh_gaussians(verts, faces[:1277], K=3, seed=11)
    # looking past the sphere: part of it is outside the view and culled (zero gradient, moments still decay)
    cam = scenes.look_at_camera((2.0, 0.4, 0.8), (0.0, 0.9, 0.0), W, H).to("cuda")
    gt_model = MeshGaussianModel.from_params(scenes.init_mesh_gaussians(verts, faces[:1277], K=3, seed=81), "cuda")
    with torch.no_grad():
        gt = render_frame(gt_model, cam, torch.ones(3, device="cuda"))[0].clamp(0, 1).contiguous()
    return p, cam, gt


def _seed_moments(opt, P, denormal):
    """Non-zero moments (a later step, not the first); `denormal`: second moments from 1e-45 (denormal) to 1e-2 and first
    moments down to 1e-40, so the tiny-argument path of the square root and denormal numerators are exercised."""
    gen = torch.Generator().manual_seed(3)
    off, n = opt.ends[-2], P * 48
    if denormal:
        v = 10.0 ** (torch.rand(n, generator=gen, dtype=torch.float64) * 43.0 - 45.0)
        m = 10.0 ** (torch.rand(n, generator=gen, dtype=torch.float64) * 38.0 - 40.0) * torch.sign(torch.randn(n, generator=gen, dtype=torch.float64))
    else:
        v = torch.rand(n, generator=gen, dtype=torch.float64) * 1e-4
        m = torch.randn(n, generator=gen, dtype=torch.float64) * 1e-3
    opt.v[off:off + n] = v.float().cuda()
    opt.m[off:off + n] = m.float().cuda()
    opt.t = 4


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("ieee", [0, 1])
@pytest.mark.parametrize("denormal", [False, True])
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_fused_sh_step_is_bit_identical_to_adam_sh_factored(degree, denormal, ieee):
    p, cam, gt = _scene()
    bg = torch.ones(3, device="cuda")
    model = MeshGaussianModel.from_params(p, "cuda", packed_features=True, active_sh_degree=degree)
    P = model._features.shape[0]
    opt = FlatAdam(mesh_model_groups(model, features_last=True), sh_factored=True)
    _seed_moments(opt, P, denormal)
    off = opt.ends[-2]
    p0 = model._features.detach().clone()
    m0 = opt.m[off:off + P * 48].clone()
    v0 = opt.v[off:off + P * 48].clone()
    m_seed = m0.clone()
    fr = NativeFrame(model, W, H)
    old = _lib.set_option("adam_sh_ieee", ieee)
    try:
        sh = opt.begin_fused_sh_step()
        fr.run(cam, gt, bg, factored=True, sh_adam=sh)       # factored: the frame also writes its colour gradient slot
        view = _lib.FrameView()
        _lib.check(_lib.lib().gms_frame_views(fr.ws.data_ptr(), P, W, H, C.byref(view)), "gms_frame_views")
        a = _lib.AdamShArgs()
        a.P, a.M, a.sh_degree, a.R = P, 16, degree, 1
        a.xyz, a.exchange, a.slot_floats, a.grad_scale = view.xyz, fr.exchange.data_ptr(), fr.exchange.shape[1], 1.0
        a.p, a.m, a.v = p0.data_ptr(), m0.data_ptr(), v0.data_ptr()
        g = opt.groups[-1]
        a.lr_dc, a.lr_rest, a.beta1, a.beta2, a.eps, a.step = g["lr0"], g["lr1"], opt.betas[0], opt.betas[1], opt.eps, opt.t
        _lib.check(_lib.lib().gms_adam_sh_factored(C.byref(a), torch.cuda.current_stream().cuda_stream), "gms_adam_sh_factored")
        torch.cuda.synchronize()
    finally:
        _lib.set_option("adam_sh_ieee", old)
    zero = (fr.exchange[0, :3 * P].view(P, 3) == 0).all(1)
    assert 0 < int(zero.sum()) < P, int(zero.sum())             # some Gaussians get a gradient, some (culled) do not
    assert torch.equal(_bits(model._features.detach()), _bits(p0))
    assert torch.equal(_bits(opt.m[off:off + P * 48]), _bits(m0))
    assert torch.equal(_bits(opt.v[off:off + P * 48]), _bits(v0))
    # rows without a gradient were stepped too: their moments decayed
    assert bool((m0.view(P, 48)[zero] != m_seed.view(P, 48)[zero]).any())
