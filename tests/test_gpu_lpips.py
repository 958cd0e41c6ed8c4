"""-m gpu: VGG16 LPIPS on the device (gms_lpips_vgg through gms_b200.lpips.Lpips), with seeded He-scaled weights written
to and loaded from the two real file formats.

1. Per view and per layer term, |native - float64| <= 8 * max over the size's views |torch float32 - float64| + 1e-7, where
   torch float32 is PyTorch's own forward with TF32 off, at 16x16, odd sizes, 800x800 and 1920x1080, for a render against
   its perturbed ground truth, unrelated images and near-identical images.
2. Identical images give exactly 0; two calls give the same bits.
3. H or W < 16, too little scratch and null pointers are refused before any launch.
4. evaluate(protocol="metrics", lpips=L) scores the 8-bit round trips bit for bit as L does, leaves per_view / mean
   unchanged, and synchronises only in its read-back.
5. cli.metrics --lpips: each per-view value is the library's LPIPS of the decoded PNGs."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lpips_oracle
from gms_b200 import _lib, io_image
from gms_b200.lpips import Lpips, scratch_bytes

pytestmark = pytest.mark.gpu

SIZES = [(16, 16), (67, 45), (135, 101), (800, 800), (1080, 1920)]      # (H, W)


@pytest.fixture(scope="module")
def weights(tmp_path_factory):
    d = tmp_path_factory.mktemp("lpips_weights")
    _, _, vgg16, lin = lpips_oracle.write_weight_files(d, seed=0)
    return str(d), Lpips.from_cache(str(d), device="cuda"), vgg16, lin


def _image(H, W, g):
    """A smooth random image in [0, 1]: low-resolution noise upsampled, plus fine grain."""
    low = torch.rand(1, 3, max(H // 8, 2), max(W // 8, 2), generator=g, device="cuda")
    img = F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False)[0]
    return (img + 0.05 * torch.rand(3, H, W, generator=g, device="cuda")).clamp(0, 1)


def _pairs(H, W):
    g = torch.Generator(device="cuda").manual_seed(H * 10007 + W)
    render = _image(H, W, g)
    perturbed = (render + 0.08 * (torch.rand(3, H, W, generator=g, device="cuda") - 0.5)).clamp(0, 1)
    unrelated = _image(H, W, g)
    near = render.clone()
    mask = torch.rand(3, H, W, generator=g, device="cuda") < 0.01
    near[mask] = (near[mask] + 1.0 / 255.0).clamp(0, 1)
    return {"perturbed": (render, perturbed), "unrelated": (render, unrelated), "near_identical": (render, near)}


def _torch_fp32(img, gt, vgg16, lin):
    cudnn, matmul = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return lpips_oracle.lpips(img, gt, vgg16, lin, dtype=torch.float32).double()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = cudnn, matmul


@pytest.mark.parametrize("H,W", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_matches_float64_within_the_float32_bound(weights, H, W):
    _, L, vgg16, lin = weights
    native, err32 = {}, {}
    for name, (img, gt) in _pairs(H, W).items():
        with torch.no_grad():
            ref = lpips_oracle.lpips(img, gt, vgg16, lin)
            t32 = _torch_fp32(img, gt, vgg16, lin)
        native[name] = (L.lpips(img, gt).double() - ref).abs()
        err32[name] = (t32 - ref).abs()
        print(f"[lpips {H}x{W} {name}] float64 {ref[5].item():.9g}: |native - f64| {native[name].max().item():.3e}, "
              f"|torch fp32 - f64| {err32[name].max().item():.3e}")
        assert torch.isfinite(ref).all() and ref[5] > 0
    bound = 8 * torch.stack(list(err32.values())).max(0).values + 1e-7
    for name, e in native.items():
        assert (e <= bound).all(), (name, e.tolist(), bound.tolist())


def test_identical_images_give_zero_and_calls_repeat_bit_for_bit(weights):
    _, L, _, _ = weights
    img, gt = _pairs(135, 101)["perturbed"]
    assert torch.equal(L.lpips(img, img.clone()), torch.zeros(6, device="cuda"))
    a, b = L.lpips(img, gt).clone(), L.lpips(img, gt).clone()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)) and a[5] > 0


def _call(L, H, W, img, gt, out, scratch, nbytes):
    a = _lib.LpipsArgs()
    a.H, a.W, a.img, a.gt, a.weights = H, W, img, gt, L.weights.data_ptr()
    a.out, a.scratch, a.scratch_bytes = out, scratch, nbytes
    return _lib.lib().gms_lpips_vgg(C.byref(a), torch.cuda.current_stream().cuda_stream)


def test_refusals_return_before_any_launch(weights):
    _, L, _, _ = weights
    img = torch.rand(3, 32, 32, device="cuda")
    out = torch.full((6,), -1.0, device="cuda")
    need = scratch_bytes(32, 32)
    assert need > 0 and scratch_bytes(15, 32) == 0 and scratch_bytes(32, 15) == 0
    s = torch.empty(need, dtype=torch.uint8, device="cuda")
    p = img.data_ptr()
    _lib.launch_count(reset=True)
    for H, W, nbytes, ptrs in [(15, 32, need, (p, p, out.data_ptr(), s.data_ptr())), (32, 15, need, (p, p, out.data_ptr(), s.data_ptr())),
                               (32, 32, need - 1, (p, p, out.data_ptr(), s.data_ptr())), (32, 32, need, (None, p, out.data_ptr(), s.data_ptr())),
                               (32, 32, need, (p, p, None, s.data_ptr())), (32, 32, need, (p, p, out.data_ptr(), None))]:
        assert _call(L, H, W, ptrs[0], ptrs[1], ptrs[2], ptrs[3], nbytes) == _lib.GMS_E_ARG
    assert _lib.launch_count() == 0
    assert (out == -1).all()
    with pytest.raises(ValueError, match="at least 16"):
        L.lpips(torch.rand(3, 15, 40, device="cuda"), torch.rand(3, 15, 40, device="cuda"))
    assert _call(L, 32, 32, p, p, out.data_ptr(), s.data_ptr(), need) == _lib.GMS_OK
    assert _lib.launch_count() > 0 and (out == 0).all()


def test_evaluate_scores_the_round_trips_in_its_single_pass(weights):
    from gms_b200.render import NativeRenderer
    from test_gpu_render_eval import BG, _model, _views
    _, L, _, _ = weights
    W, H = 256, 256
    p, cams, gts8 = _views(4, W, H)
    gts = [io_image.to_device_float(t).clone() for t in gts8]
    bg = torch.tensor(BG, device="cuda")
    model = _model(p)
    plain = NativeRenderer(model, W, H).evaluate(cams, gts, bg, protocol="metrics")
    assert plain.lpips is None
    r = NativeRenderer(model, W, H)
    r.evaluate(cams, gts, bg, protocol="metrics")         # learns every view's N: the next pass is sync-free
    torch.cuda.synchronize()
    # evaluate's read-back: one stream synchronise, then per_view's copy to the host; anything else that synchronises
    # raises under sync debug mode "error"
    relaxed = []

    def relax(fn, what):
        def call(*a, **k):
            relaxed.append(what)
            torch.cuda.set_sync_debug_mode(0)
            try:
                return fn(*a, **k)
            finally:
                torch.cuda.set_sync_debug_mode("error")
        return call

    mp = pytest.MonkeyPatch()
    mp.setattr(torch.cuda.Stream, "synchronize", relax(torch.cuda.Stream.synchronize, "stream"))
    mp.setattr(torch.Tensor, "cpu", relax(torch.Tensor.cpu, "cpu"))
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = r.evaluate(cams, gts, bg, protocol="metrics", lpips=L)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        mp.undo()
    assert relaxed == ["stream", "cpu"], relaxed
    assert res.rerun == []
    assert torch.equal(res.per_view.view(torch.int64), plain.per_view.view(torch.int64))
    assert torch.equal(res.mean.view(torch.int64), plain.mean.view(torch.int64))
    assert res.lpips.dtype == torch.float32 and res.lpips.shape == (4,)
    for v, cam in enumerate(cams):
        image = r.render(cam, bg)[0]
        q = io_image.to_device_float(io_image.quantize(image).view(H, W, 3))
        g = io_image.to_device_float(io_image.quantize(gts[v]).view(H, W, 3))
        want = L.lpips(q, g)[5].cpu()
        assert torch.equal(res.lpips[v:v + 1].view(torch.int32), want.view(1).view(torch.int32)), v
    with pytest.raises(ValueError, match="metrics"):
        r.evaluate(cams, gts, bg, protocol="training_report", lpips=L)


def test_metrics_cli_lpips_matches_the_library_on_the_pngs(weights, tmp_path):
    from gms_b200.cli import metrics as cli_metrics
    from gms_b200.render import NativeRenderer
    from test_gpu_render_eval import BG, _model, _views
    wdir, L, _, _ = weights
    W, H = 256, 256
    p, cams, gts8 = _views(3, W, H)
    r = NativeRenderer(_model(p), W, H)
    d = tmp_path / "model" / "test" / "ours_30"
    os.makedirs(d / "renders_gs_flat")
    os.makedirs(d / "gt")
    for i, cam in enumerate(cams):
        io_image.save_image(r.render(cam, torch.tensor(BG, device="cuda"))[0], str(d / "renders_gs_flat" / f"{i:05d}.png"))
        io_image.save_image(io_image.to_device_float(gts8[i]), str(d / "gt" / f"{i:05d}.png"))
    model = str(tmp_path / "model")
    res = cli_metrics.main(["-m", model, "--gs_type", "gs_flat", "--quiet", "--lpips", "--lpips_weights", wdir])[model]
    pv = res["per_view"]["ours_30"]
    assert list(pv) == ["SSIM", "PSNR", "LPIPS"] and list(res["results"]["ours_30"]) == ["SSIM", "PSNR", "LPIPS"]
    for name, got in pv["LPIPS"].items():
        x, y = (io_image.to_device_float(io_image.load_image_u8(str(d / sub / name)).cuda()) for sub in ("renders_gs_flat", "gt"))
        assert got == L.lpips(x, y)[5].item(), name
    lp = np.array(list(pv["LPIPS"].values()), dtype=np.float32)
    assert res["results"]["ours_30"]["LPIPS"] == torch.tensor(lp).mean().item()
    with open(os.path.join(model, "results_gs_flat.json")) as f:
        assert list(json.load(f)["ours_30"]) == ["SSIM", "PSNR", "LPIPS"]
