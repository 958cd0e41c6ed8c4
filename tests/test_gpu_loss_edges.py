"""-m gpu: the fused L1+SSIM loss (gms_l1_ssim_loss: k_ssim_stats -> k_loss_finalize -> k_ssim_grad) and the image-metric
kernel (gms_image_metrics: k_image_metrics<Q>) against the float64 restatement of tests/loss_oracle.py, pixel by pixel, at
tile, halo and image edges.

1. Impulse lattices: dL/dx is nonzero exactly on the 21 x 21 box around each impulse (a missing halo row, column or corner
   tap in either kernel zeroes part of a box's outer ring), and within K * bound inside the boxes.
2. Sizes that miss the 32-pixel tile by less than the 5-pixel halo, 1 x N and N x 1, 1080p and 4K (n > 2^24), times six
   contents (uniform, 30 % exact ties, a matched white background, renders above 1, a u8 ground truth, all zeros):
   every element of dL/dx within K * bound; loss, L1 and SSIM within K * a bound derived from the kernel's summation.
3. lambda = 0 gives fl(1/n) sign(x - y) bit for bit (0 on ties); lambda = 1 holds the SSIM part alone to the bound.
4. The C ABI's optional pointers: a device dL_dloss scales the gradient bit for bit; dL_dimg = NULL writes nothing.
5. gms_image_metrics for both protocols against the restatement's summation bound, at the quantiser's rounding edges, and
   deterministic."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import aten_reference
import loss_oracle as lo
from gms_b200 import _lib
from gms_b200.metrics import image_metrics
from metrics_restated import transform

pytestmark = pytest.mark.gpu

_ref_cache = {}


def _case(H, W, content):
    return lo.make_case(H, W, content, seed=31 * H + W)


def _ref(key, x, y, lam):
    """loss64 with its bound, in float64 on the GPU, cached per case."""
    k = key + (lam,)
    if k in _ref_cache:
        return _ref_cache[k]
    r = lo.loss64(x.cuda(), y.cuda(), lam, bound=True)
    r = {n: r[n] for n in ("loss", "l1", "ssim", "grad", "grad_bound", "m", "m_bound")} | \
        {"sums_bound": lo.loss_sums_bound(x.cuda(), y.cuda(), r, lam)}
    if x.numel() <= 1 << 22:                          # 1080p and 4K references are not kept
        _ref_cache[k] = r
    return r


def _loss(x, y, lam, up=None, grad=True, scratch_fill=None):
    """gms_l1_ssim_loss through the raw C ABI.  Returns (loss[3], dL/dimg or None, scratch)."""
    L = _lib.lib()
    x, y = x.cuda().contiguous(), y.cuda().contiguous()
    Cn, H, W = x.shape
    nb = C.c_size_t()
    _lib.check(L.gms_loss_scratch_bytes(Cn, H, W, C.byref(nb)), "gms_loss_scratch_bytes")
    scratch = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    if scratch_fill is not None:
        scratch.fill_(scratch_fill)
    out = torch.empty(3, device="cuda")
    dimg = torch.empty_like(x) if grad else None
    upt = torch.tensor([up], dtype=torch.float32, device="cuda") if up is not None else None
    a = _lib.LossArgs(Cn, H, W, x.data_ptr(), y.data_ptr(), float(lam), upt.data_ptr() if upt is not None else None,
                      out.data_ptr(), dimg.data_ptr() if grad else None, scratch.data_ptr(), nb.value)
    _lib.check(L.gms_l1_ssim_loss(C.byref(a), torch.cuda.current_stream().cuda_stream), "gms_l1_ssim_loss")
    torch.cuda.synchronize()
    return out.cpu().double(), dimg, scratch


def _check_sums(what, got, r):
    for i, k in enumerate(("loss", "l1", "ssim")):
        err, b = abs(float(got[i]) - r[k]), r["sums_bound"][k]
        print(f"[loss sums] {what} {k}: err {err:.3e} bound {b:.3e}")
        assert err <= lo.K * b, (what, k, float(got[i]), r[k], b)


def _grad_ratio(g, r):
    return lo.ratio((g.double() - r["grad"]).abs(), r["grad_bound"])


# ---- 1. impulse lattices
@pytest.mark.parametrize("name", list(lo.lattice_cases()))
def test_lattice_gradient_support_is_exact_and_values_are_bounded(name):
    H, W, rows, cols = lo.lattice_cases()[name]
    x, y, support = lo.lattice(H, W, rows, cols, seed=H + W)
    r = _ref((name, "lattice"), x, y, 0.2)
    out, g, _ = _loss(x, y, 0.2)
    nz = (g != 0).cpu()
    stray, holes = int((nz & ~support).sum()), int((~nz & support).sum())
    q = _grad_ratio(g, r)
    print(f"[loss lattice] {name}: stray nonzeros {stray}, zeros inside boxes {holes} of {nz.numel()}; err / bound {q:.3f}")
    assert stray == 0 and holes == 0
    assert q <= lo.K
    _check_sums(name, out, r)


# ---- 2. size x content sweep at lambda = 0.2
_worst = {}


@pytest.mark.parametrize("H,W", lo.SWEEP_SIZES + lo.LARGE_SIZES)
def test_gradient_and_sums_within_the_bound(H, W):
    for content in lo.CONTENTS:
        x, y = _case(H, W, content)
        r = _ref((H, W, content), x, y, 0.2)
        out, g, _ = _loss(x, y, 0.2)
        q = _grad_ratio(g, r)
        _worst[content] = max(_worst.get(content, 0.0), q)
        print(f"[loss sweep] {W}x{H} {content}: err / bound {q:.3f} (worst {content} so far {_worst[content]:.3f})")
        assert q <= lo.K, (H, W, content, q)
        _check_sums(f"{W}x{H} {content}", out, r)


def test_flat_tie_gradient_against_fp32_aten():
    """A matched white background (x = y = 1 away from a textured patch): the float64 gradient there is 0.  Reports how far
    the kernel's and fp32 ATen's gradients stray from 0 there, in units of 1/n, and holds both to the bound."""
    H, W = 201, 333
    x, y = _case(H, W, "white")
    r = _ref((H, W, "white"), x, y, 0.2)
    _, g, _ = _loss(x, y, 0.2)
    a = x.clone().requires_grad_(True)
    aten_reference.training_loss(a, y, 0.2).backward()
    flat = torch.zeros(H, W, dtype=torch.bool)
    flat[:H // 3 - 10, :] = True                      # more than 10 px (two filter radii) above the patch
    n = x.numel()
    k_flat = float(g.cpu()[:, flat].abs().max()) * n
    a_flat = float(a.grad[:, flat].abs().max()) * n
    b_flat = float(r["grad_bound"].cpu()[:, flat].max()) * n
    print(f"[loss flat ties] max |g| * n over the flat region: kernel {k_flat:.3e}, fp32 ATen (CPU) {a_flat:.3e}, "
          f"float64 {float(r['grad'].cpu()[:, flat].abs().max()) * n:.1e}, bound {b_flat:.3e}")
    assert k_flat <= lo.K * b_flat and a_flat <= lo.K * b_flat


# ---- 3. lambda
@pytest.mark.parametrize("H,W", [(1, 69), (69, 1), (31, 32), (33, 37), (65, 69), (1080, 1920)])
def test_lambda_zero_is_the_l1_subgradient_bit_for_bit(H, W):
    for content in ("ties30", "white", "zeros"):
        x, y = _case(H, W, content)
        out, g, _ = _loss(x, y, 0.0)
        inv_n = np.float32(1.0) / np.float32(x.numel())
        want = torch.sign(x - y) * torch.tensor(inv_n)
        assert torch.equal(g.cpu(), want), (H, W, content)
        assert int((g.cpu()[x == y] != 0).sum()) == 0


@pytest.mark.parametrize("H,W", [(6, 11), (33, 37), (65, 69), (201, 333)])
def test_lambda_one_holds_the_ssim_part_alone_to_the_bound(H, W):
    for content in ("uniform", "white", "hdr", "u8"):
        x, y = _case(H, W, content)
        r = _ref((H, W, content), x, y, 1.0)
        out, g, _ = _loss(x, y, 1.0)
        q = _grad_ratio(g, r)
        print(f"[loss lambda=1] {W}x{H} {content}: err / bound {q:.3f}")
        assert q <= lo.K
        _check_sums(f"lambda=1 {W}x{H} {content}", out, r)


# ---- 4. the C ABI's optional pointers
@pytest.mark.parametrize("H,W", [(33, 37), (201, 333)])
def test_upstream_scales_the_gradient_bit_for_bit(H, W):
    x, y = _case(H, W, "ties30")
    out1, g1, _ = _loss(x, y, 0.2)
    for up in (3.0, -0.5, 0.0):
        out, g, _ = _loss(x, y, 0.2, up=up)
        assert torch.equal(g, g1 * up), up
        r = _ref((H, W, "ties30"), x, y, 0.2)
        _check_sums(f"up={up}", out, r)          # the loss itself is not scaled


@pytest.mark.parametrize("H,W", [(33, 37), (201, 333)])
def test_null_gradient_pointer_writes_no_gradient(H, W):
    x, y = _case(H, W, "uniform")
    out_g, _, _ = _loss(x, y, 0.2)
    out, _, scratch = _loss(x, y, 0.2, grad=False, scratch_fill=0xA5)
    base = (256 - scratch.data_ptr() % 256) % 256
    s = scratch.cpu()
    assert bool((s[:base] == 0xA5).all()) and bool((s[base + 8:] == 0xA5).all())   # only acc[0..1] was written
    r = _ref((H, W, "uniform"), x, y, 0.2)
    for i, k in enumerate(("loss", "l1", "ssim")):    # two runs of the same sums: only the atomics' order differs
        assert abs(float(out[i]) - float(out_g[i])) <= 2 * r["sums_bound"][k], k


# ---- 5. image metrics
def _check_metrics(what, got, vals, bounds):
    got = [float(v) for v in got]
    for k, name in enumerate(("l1", "ssim", "psnr", "psnr_c")):
        if math.isinf(vals[k]):
            assert math.isinf(got[k]) and got[k] > 0, (what, name)
            continue
        err = abs(got[k] - vals[k])
        print(f"[metrics] {what} {name}: err {err:.3e} bound {bounds[k]:.3e}")
        assert err <= lo.K * bounds[k], (what, name, got[k], vals[k], bounds[k])


@pytest.mark.parametrize("protocol", ["training_report", "metrics"])
@pytest.mark.parametrize("H,W", [(1, 69), (69, 1), (6, 11), (27, 31), (33, 37), (38, 63), (65, 69), (1080, 1920)])
def test_image_metrics_within_the_summation_bound_and_deterministic(H, W, protocol):
    for content in lo.CONTENTS:
        x, y = _case(H, W, content)
        a = image_metrics(x.cuda(), y.cuda(), protocol).cpu()
        b = image_metrics(x.cuda(), y.cuda(), protocol).cpu()
        assert torch.equal(a.view(torch.int64), b.view(torch.int64))
        vals, bounds = lo.metrics64_bound(x.cuda(), y.cuda(), protocol)
        _check_metrics(f"{protocol} {W}x{H} {content}", a, vals, bounds)


def test_image_metrics_quantiser_rounding_edges():
    """Values at k/255 and (k +- 0.5)/255, each +- 1 ulp: the kernel's byte must be the byte of ATen's mul(255).add(0.5)
    .clamp(0, 255).to(uint8).  Against the ATen-quantised copy of itself, any differing byte makes L1 > 0."""
    k = np.arange(256, dtype=np.float64)
    base = np.concatenate([k / 255, (k + 0.5) / 255, (k - 0.5) / 255]).astype(np.float32)
    vals = np.concatenate([base, np.nextafter(base, np.float32(np.inf)), np.nextafter(base, np.float32(-np.inf)),
                           np.array([-1.0, -0.0, 1.5, 255.0, 1.0 + 2 ** -23], dtype=np.float32)])
    g = torch.Generator().manual_seed(4)
    flat = torch.from_numpy(np.resize(vals, 3 * 32 * 40))          # every value at least once, in a shuffled layout
    img = flat[torch.randperm(flat.numel(), generator=g)].reshape(3, 32, 40).contiguous()
    q = transform(img, "metrics")                    # ATen's bytes / 255
    got = image_metrics(img.cuda(), q.cuda(), "metrics").cpu()
    assert float(got[0]) == 0.0 and got[2] == math.inf, [float(v) for v in got]
    vals_, bounds = lo.metrics64_bound(img.cuda(), torch.zeros_like(img).cuda(), "metrics")
    _check_metrics("quantiser edges vs 0", image_metrics(img.cuda(), torch.zeros_like(img).cuda(), "metrics").cpu(), vals_, bounds)
