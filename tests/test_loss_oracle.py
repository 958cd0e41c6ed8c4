"""CPU: the float64 restatement of the fused loss (tests/loss_oracle.py) against the ATen restatement and the reference's
own loss fixture, and its per-pixel bound against what fp32 ATen arithmetic actually does."""
import os

import numpy as np
import pytest
import torch

import aten_reference
import loss_oracle as lo
from metrics_restated import metrics64


def _aten(x, y, lam, up=1.0):
    a = x.clone().requires_grad_(True)
    loss = aten_reference.training_loss(a, y.to(x.dtype), lam)
    (loss * up).backward()
    return float(loss), a.grad


@pytest.mark.parametrize("lam,up", [(0.2, 1.0), (0.0, 3.0), (1.0, -0.5), (0.7, 1.0)])
@pytest.mark.parametrize("H,W", [(45, 70), (1, 37), (33, 1), (64, 65)])
def test_loss64_equals_aten_in_float64(H, W, lam, up, monkeypatch):
    """Same maths, same window: ATen's 2-D window is replaced by the outer product of the kernel's taps in double, and the
    SSIM constants are the exact ones aten_reference uses."""
    x, y = lo.make_case(H, W, "ties30", H * W)
    g = torch.tensor(lo.WIN, dtype=torch.float64)
    monkeypatch.setitem(aten_reference._window_cache, (11, 3, "cpu", torch.float64),
                        (g[:, None] * g[None, :]).expand(3, 1, 11, 11).contiguous())
    l_ref, g_ref = _aten(x.double(), y.double(), lo._f32(lam), lo._f32(up))
    r = lo.loss64(x, y, lam, up, c1=0.01 ** 2, c2=0.03 ** 2)
    assert abs(r["loss"] - l_ref) <= 1e-12 * abs(l_ref)
    assert float((r["grad"] - g_ref).abs().max()) <= 1e-10 * float(g_ref.abs().max())


def test_loss64_reproduces_the_reference_fixture(golden_dir):
    """tests/golden/loss.npz: the reference's utils/loss_utils.py in fp32 (its own window and fp32 arithmetic)."""
    d = np.load(os.path.join(golden_dir, "loss.npz"))
    x, y = torch.from_numpy(d["img"]), torch.from_numpy(d["gt"])
    r = lo.loss64(x, y, 0.2, bound=True)
    b = lo.loss_sums_bound(x, y, r, 0.2)
    for k in ("loss", "l1", "ssim"):
        assert abs(r[k] - float(d[k])) <= lo.K * b[k] + 1e-7, (k, r[k], float(d[k]), b[k])
    q = lo.ratio((torch.from_numpy(d["grad"]).double() - r["grad"]).abs(), r["grad_bound"])
    print(f"[loss64] reference fixture: gradient err / bound {q:.3f}")
    assert q <= lo.K


_worst = {}


@pytest.mark.parametrize("content", lo.CONTENTS)
@pytest.mark.parametrize("H,W", lo.SWEEP_SIZES + [(1080, 1920)])
def test_fp32_aten_stays_within_the_bound(H, W, content):
    """The bound models fp32 arithmetic: fp32 ATen (121-tap 2-D convolutions, another factorisation, its own window) stays
    inside K * bound, per element, at the sizes and contents the GPU sweep uses."""
    if (H, W) == (1080, 1920) and content not in ("uniform", "white"):
        pytest.skip("1080p: two contents are enough on the CPU")
    x, y = lo.make_case(H, W, content, 7 * H + W)
    r = lo.loss64(x, y, 0.2, bound=True)
    l32, g32 = _aten(x, y, 0.2)
    q = lo.ratio((g32.double() - r["grad"]).abs(), r["grad_bound"])
    _worst[content] = max(_worst.get(content, 0.0), q)
    print(f"[aten fp32] {W}x{H} {content}: err / bound {q:.3f} (worst for {content} so far {_worst[content]:.3f})")
    assert q <= lo.K


@pytest.mark.parametrize("name", list(lo.lattice_cases()))
def test_lattice_support_is_exact_in_float64_and_fp32_aten(name):
    """dL/dx is nonzero exactly on the 21 x 21 boxes around the impulses, in float64 and in fp32 ATen alike."""
    H, W, rows, cols = lo.lattice_cases()[name]
    x, y, support = lo.lattice(H, W, rows, cols, seed=H + W)
    r = lo.loss64(x, y, 0.2, bound=True)
    _, g32 = _aten(x, y, 0.2)
    for what, g in (("float64", r["grad"]), ("fp32 aten", g32)):
        nz = g != 0
        assert int((nz & ~support).sum()) == 0 and int((~nz & support).sum()) == 0, what
    assert lo.ratio((g32.double() - r["grad"]).abs(), r["grad_bound"]) <= lo.K


def test_flat_tie_gradient_is_zero_in_float64_and_bounded_away_from_zero():
    """x = y = 1 (a matched white background): the float64 gradient is 0 up to double rounding inside the flat region,
    while the bound there stays positive (it comes from B2 = C2's conditioning)."""
    x, y = lo.make_case(96, 96, "white", 3)
    r = lo.loss64(x, y, 0.2, bound=True)
    n = x.numel()
    flat = torch.zeros(96, 96, dtype=torch.bool)
    flat[:10, :] = True                               # more than 10 px from the patch (rows 32..63)
    g, b = r["grad"][:, flat], r["grad_bound"][:, flat]
    assert float(g.abs().max()) * n <= 1e-12
    assert float(b.min()) > 0


@pytest.mark.parametrize("protocol", ["training_report", "metrics"])
def test_metrics_restatement_with_the_kernel_window_matches_metrics64(protocol):
    """Only the window differs: metrics64 uses exact taps, the kernel fp32 ones (their sum is 1 + 4.4e-8), which moves SSIM
    by up to a few 1e-7 where clamping flattens the image."""
    x, y = lo.make_case(65, 69, "hdr", 11)
    vals, bounds = lo.metrics64_bound(x, y, protocol)
    ref = metrics64(x, y, protocol)
    for k in range(4):
        assert abs(vals[k] - ref[k]) <= (1e-6 if k == 1 else 1e-12) * max(1.0, abs(ref[k])), (k, vals[k], ref[k])
        assert bounds[k] > 0
