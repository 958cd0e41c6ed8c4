"""Float64 restatement of the fused training loss (csrc/gms_loss.cuh: k_ssim_stats -> k_loss_finalize -> k_ssim_grad) and of
the image-metric kernel k_image_metrics<Q>, with a per-pixel first-order bound on how far fp32 arithmetic of the same
operations may stray from it -- TEST INFRASTRUCTURE.

The restatement filters with the kernel's own window (ssim_window(): fp32 taps, promoted to double), takes lambda and the
SSIM constants as the fp32 values the kernel sees, and computes dL/dx analytically in the kernel's factorisation
    dL/dx = up * ( c_ssim * [G*d_mu + 2x G*d_ess + y G*d_exy] + c_l1 * sign(x - y) ),  c_ssim = -lambda/n, c_l1 = (1-lambda)/n
so that a comparison measures only the kernel's arithmetic.

The bound (u = 2^-24, GAMMA = GAMMA_C * u; each item is first order in u):
  1. each filtered moment (mu_x, mu_y, E[x^2+y^2], E[xy]) is off by at most GAMMA * G*(|x|, |y|, x^2+y^2, |xy|): two 11-tap
     fma chains and one product per tap;
  2. the SSIM map and its three partials carry that through the sensitivities of the elementwise pixel function (four
     float64 forward-mode derivatives), plus a running-error bound of the pixel function's own roundings, u |value| per
     operation;
  3. the gradient: |c_ssim| (G*dd_mu + 2|x| G*dd_ess + |y| G*dd_exy) + GAMMA |c_ssim| (G*|d_mu| + 2|x| G*|d_ess| + |y| G*|d_exy|)
     plus the epilogue's roundings;
  4. the L1 term needs none: sign(fl(x - y)) = sign(x - y) exactly; only its fp32 coefficient is rounded.
Where the float64 gradient is 0 (flat tie regions) the bound still comes out positive, from the conditioning of
B2 = sigma_x^2 + sigma_y^2 + C2 in step 2."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24
GAMMA_C = 8.0                   # two 11-tap fma chains + one product: a first-order running-error estimate, not the worst case
GAMMA = GAMMA_C * U
K = 4.0                         # every kernel and fp32 ATen result is held to K * bound
RED_TREE = 11                   # k_ssim_stats / k_image_metrics: 4 values per thread, 5 shuffle levels, 3 levels over 8 warps
TILE, RADIUS = 32, 5


def _f32(v: float) -> float:
    return float(np.float32(v))


C1_F32 = float(np.float32(0.01) * np.float32(0.01))      # 0.01f * 0.01f, as the kernel folds it
C2_F32 = float(np.float32(0.03) * np.float32(0.03))


def ssim_window() -> list:
    """gms_kernels.cu ssim_window(): exp in double rounded to fp32, summed in fp32 in order, each tap divided in fp32."""
    g = [np.float32(math.exp(-float((k - 5) * (k - 5)) / (2.0 * 1.5 * 1.5))) for k in range(11)]
    s = np.float32(0.0)
    for v in g:
        s = np.float32(s + v)
    return [float(np.float32(v / s)) for v in g]


WIN = ssim_window()


def filt(t: torch.Tensor, win=WIN) -> torch.Tensor:
    """Separable zero-padded 11-tap filter of [..., H, W], horizontal pass first, in t's dtype."""
    H, W = t.shape[-2:]
    p = F.pad(t, (RADIUS, RADIUS, RADIUS, RADIUS))
    h = win[0] * p[..., :, 0:W]
    for k in range(1, 11):
        h = h + win[k] * p[..., :, k:k + W]
    v = win[0] * h[..., 0:H, :]
    for k in range(1, 11):
        v = v + win[k] * h[..., k:k + H, :]
    return v


def pixel(mu1, mu2, ess, exy, c1=C1_F32, c2=C2_F32):
    """gms_ssim_pixel and k_ssim_stats' three partials: (SSIM map, dm/dmu_x, dm/dE[x^2+y^2], dm/dE[xy])."""
    mu1s, mu2s, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    A1, A2 = 2 * mu12 + c1, 2 * (exy - mu12) + c2
    B1, B2 = mu1s + mu2s + c1, (ess - mu1s - mu2s) + c2
    r1, r2 = 1 / B1, 1 / B2
    inv = r1 * r2
    m = A1 * A2 * inv
    return m, 2 * mu2 * (A2 - A1) * inv - m * 2 * mu1 * (r1 - r2), -m * r2, 2 * A1 * inv


def pixel_rounding(mu1, mu2, ess, exy, c1=C1_F32, c2=C2_F32):
    """Running-error bound, in units of u, of pixel()'s own fp32 roundings from exact inputs (Wilkinson: each operation adds
    u |result|, and carries its operands' bounds through its partial derivatives).  Contracting a pair into an fma only
    removes a rounding, so the bound holds for either code generation."""
    a = torch.abs
    mu1s, mu2s, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    e1s, e2s, e12 = a(mu1s), a(mu2s), a(mu12)
    s12 = exy - mu12; es12 = e12 + a(s12)
    A1 = 2 * mu12 + c1; eA1 = 2 * e12 + a(A1)
    A2 = 2 * s12 + c2; eA2 = 2 * es12 + a(A2)
    t = mu1s + mu2s; et = e1s + e2s + a(t)
    B1 = t + c1; eB1 = et + a(B1)
    t1 = ess - mu1s; e = e1s + a(t1)
    t2 = t1 - mu2s; e = e + e2s + a(t2)
    B2 = t2 + c2; eB2 = e + a(B2)
    r1, r2 = 1 / B1, 1 / B2
    er1, er2 = eB1 * r1 * r1 + a(r1), eB2 * r2 * r2 + a(r2)
    inv = r1 * r2; einv = er1 * a(r2) + er2 * a(r1) + a(inv)
    p = A1 * A2; ep = eA1 * a(A2) + eA2 * a(A1) + a(p)
    m = p * inv; em = ep * a(inv) + einv * a(p) + a(m)
    d2 = A2 - A1; ed2 = eA2 + eA1 + a(d2)
    t3 = 2 * mu2 * d2; e3 = 2 * a(mu2) * ed2 + a(t3)
    t4 = t3 * inv; e4 = e3 * a(inv) + einv * a(t3) + a(t4)
    s1 = m * 2 * mu1; es1 = em * 2 * a(mu1) + a(s1)
    s2 = r1 - r2; es2 = er1 + er2 + a(s2)
    s3 = s1 * s2; es3 = es1 * a(s2) + es2 * a(s1) + a(s3)
    d_mu = t4 - s3; edmu = e4 + es3 + a(d_mu)
    d_ess = -m * r2; edss = em * a(r2) + er2 * a(m) + a(d_ess)
    d_exy = 2 * A1 * inv; edxy = 2 * eA1 * a(inv) + 2 * a(A1) * einv + a(d_exy)
    return em, edmu, edss, edxy


def _moments(x, y):
    return filt(x), filt(y), filt(x * x + y * y), filt(x * y)


def _pixel_bound(x, y, mom, c1, c2):
    """Per-pixel bound on (m, d_mu, d_ess, d_exy) from the moments' errors (step 1) and the pixel function's roundings (step 2)."""
    dmom = (GAMMA * filt(x.abs()), GAMMA * filt(y.abs()), GAMMA * filt(x * x + y * y), GAMMA * filt((x * y).abs()))
    f = lambda *q: pixel(*q, c1=c1, c2=c2)
    out = [U * e for e in pixel_rounding(*mom, c1=c1, c2=c2)]
    for k in range(4):
        tang = tuple(torch.ones_like(q) if j == k else torch.zeros_like(q) for j, q in enumerate(mom))
        _, sens = torch.func.jvp(f, tuple(mom), tang)
        out = [o + s.abs() * dmom[k] for o, s in zip(out, sens)]
    return out


def loss64(x: torch.Tensor, y: torch.Tensor, lam: float, up: float = 1.0, bound: bool = False, c1=C1_F32, c2=C2_F32, win=WIN):
    """[C,H,W] render x and ground truth y (any float dtype and device; computed in float64 on that device).  Returns a dict:
    loss, l1, ssim (floats); mu1, mu2, ess, exy (moments), m, d_mu, d_ess, d_exy (SSIM map and partials), grad = dL/dx.
    With bound=True also: grad_bound (per element), m_bound (per pixel), c_ssim, c_l1.  lam and up are taken as the fp32
    values the kernel sees."""
    x, y = x.detach().double(), y.detach().double()
    lam, up = _f32(lam), _f32(up)
    n = x.numel()
    f = (lambda t: filt(t, win))
    mom = (f(x), f(y), f(x * x + y * y), f(x * y))
    m, d_mu, d_ess, d_exy = pixel(*mom, c1=c1, c2=c2)
    c_ssim, c_l1 = -lam / n, (1.0 - lam) / n
    d = x - y
    sgn = torch.sign(d)
    g_ssim = f(d_mu) + 2 * x * f(d_ess) + y * f(d_exy)
    grad = up * (c_ssim * g_ssim + c_l1 * sgn)
    l1, ss = float(d.abs().sum()) / n, float(m.sum()) / n
    r = dict(loss=(1 - lam) * l1 + lam * (1 - ss), l1=l1, ssim=ss, mu1=mom[0], mu2=mom[1], ess=mom[2], exy=mom[3], m=m,
             d_mu=d_mu, d_ess=d_ess, d_exy=d_exy, grad=grad, c_ssim=c_ssim, c_l1=c_l1)
    if bound:
        bm, bmu, bss, bxy = _pixel_bound(x, y, mom, c1, c2)
        ax, ay = x.abs(), y.abs()
        prop = f(bmu) + 2 * ax * f(bss) + ay * f(bxy)
        filt_abs = f(d_mu.abs()) + 2 * ax * f(d_ess.abs()) + ay * f(d_exy.abs())
        # epilogue: g0 + 2x g1 + y g2 (3 roundings), * c_ssim, + c_l1 sgn, * up; c_ssim and c_l1 are themselves fp32
        epi = 6 * U * (abs(c_ssim) * filt_abs + abs(c_l1) * sgn.abs())
        r["grad_bound"] = abs(up) * (abs(c_ssim) * (prop + GAMMA * filt_abs) + epi)
        r["m_bound"] = bm
    return r


def sum_bound(per_item_abs: torch.Tensor, per_item_err: torch.Tensor | None, n_blocks: int) -> float:
    """Bound on the fp32 sum of many per-pixel values as k_ssim_stats forms it: per-value errors, a 256-thread block tree
    (RED_TREE roundings deep), then n_blocks float atomics in any order (each rounds at most u times the running sum, which is
    at most the sum of the magnitudes)."""
    s = float(per_item_abs.sum())
    e = float(per_item_err.sum()) if per_item_err is not None else 0.0
    return e + (RED_TREE + max(n_blocks - 1, 0)) * U * s


def n_tiles(H: int, W: int) -> int:
    return ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)


def loss_sums_bound(x: torch.Tensor, y: torch.Tensor, r: dict, lam: float) -> dict:
    """Bounds on k_loss_finalize's loss, L1 and SSIM (r = loss64(..., bound=True))."""
    x, y = x.detach().double(), y.detach().double()
    Cn, H, W = x.shape
    n, nb = x.numel(), Cn * n_tiles(H, W)
    lam = _f32(lam)
    d = (x - y).abs()
    b_l1 = sum_bound(d, U * d, nb) / n + 2 * U * r["l1"]                       # fl(x - y), the sums, * fl(1/n)
    b_ss = sum_bound(r["m"].abs(), r["m_bound"], nb) / n + 2 * U * abs(r["ssim"])
    b_loss = (1 - lam) * b_l1 + lam * b_ss + 4 * U * ((1 - lam) * r["l1"] + lam * (1 + abs(r["ssim"])))
    return dict(loss=b_loss, l1=b_l1, ssim=b_ss)


# ---- k_image_metrics<Q>: both images through the protocol's transform, then per-tile fp32 block sums, added in double
def metrics64_bound(img: torch.Tensor, gt: torch.Tensor, protocol: str) -> tuple:
    """(values, bounds) of L1, SSIM, PSNR, mean per-channel PSNR, restated with the kernel's window.  The transform is
    metrics_restated.transform (fp32, as the reference evaluates it); the kernel must reproduce it bit for bit."""
    from metrics_restated import transform
    dev = img.device
    x, y = transform(img, protocol).double().to(dev), transform(gt, protocol).double().to(dev)
    Cn, H, W = x.shape
    n = x.numel()
    mom = _moments(x, y)
    m = pixel(*mom)[0]
    bm = _pixel_bound(x, y, mom, C1_F32, C2_F32)[0]
    d = x - y
    ad, sq = d.abs(), d * d
    l1, ss, mse = float(ad.sum()) / n, float(m.sum()) / n, float(sq.sum()) / n
    # per-tile sums: fl(x - y) (u), fmaf(d, d, s) (2u on d^2), the block tree; then double adds (negligible, 1e-15 relative)
    b_l1 = (1 + RED_TREE) * U * l1 + 1e-15 * l1
    b_ss = float(bm.sum()) / n + RED_TREE * U * float(m.abs().sum()) / n + 1e-15 * abs(ss)
    b_mse = (2 + RED_TREE) * U * mse
    mse_c = sq.reshape(Cn, -1).mean(1)
    psnr = lambda v: -10.0 * math.log10(v) if v > 0 else math.inf
    dpsnr = lambda v, b: 10.0 / math.log(10.0) * b / v + 1e-12 if v > 0 else 0.0
    vals = [l1, ss, psnr(mse), sum(psnr(float(v)) for v in mse_c) / Cn]
    bounds = [b_l1, b_ss, dpsnr(mse, b_mse), sum(dpsnr(float(v), (2 + RED_TREE) * U * float(v)) for v in mse_c) / Cn]
    return vals, bounds


# ---- inputs at the edges where the kernels can go wrong
SIZE_SET = (1, 2, 5, 6, 11, 26, 27, 31, 32, 33, 37, 38, 63, 64, 65, 69)
SWEEP_SIZES = [(1, 69), (69, 1), (1, 1), (2, 5), (5, 2), (1, 33), (33, 1), (6, 11), (11, 26), (26, 27), (27, 31), (31, 32),
               (32, 33), (33, 37), (37, 38), (38, 63), (63, 64), (64, 65), (65, 69), (69, 6), (32, 32), (64, 64)]
LARGE_SIZES = [(1080, 1920), (2160, 3840)]
CONTENTS = ("uniform", "ties30", "white", "hdr", "u8", "zeros")


def make_case(H: int, W: int, content: str, seed: int, C: int = 3) -> tuple:
    """fp32 [C,H,W] (render, ground truth) pairs:
    uniform   both U[0,1)
    ties30    a noisy copy of the ground truth with 30 % of its elements equal to it exactly
    white     x = y = 1.0 (a white background the render matches) around a textured patch in the middle third
    hdr       renders in [0, 3) (colours are not clamped above) against a [0, 1) ground truth
    u8        a ground truth of whole bytes / 255 and a render near it
    zeros     both 0"""
    g = torch.Generator().manual_seed(seed)
    if content == "uniform":
        return torch.rand(C, H, W, generator=g), torch.rand(C, H, W, generator=g)
    if content == "ties30":
        y = torch.rand(C, H, W, generator=g)
        x = (y + 0.1 * torch.randn(C, H, W, generator=g)).clamp(0, 1)
        tie = torch.rand(C, H, W, generator=g) < 0.3
        x[tie] = y[tie]
        return x, y
    if content == "white":
        x, y = torch.ones(C, H, W), torch.ones(C, H, W)
        h0, w0 = H // 3, W // 3
        h1, w1 = max(h0 + 1, 2 * H // 3), max(w0 + 1, 2 * W // 3)
        x[:, h0:h1, w0:w1] = torch.rand(C, h1 - h0, w1 - w0, generator=g)
        y[:, h0:h1, w0:w1] = torch.rand(C, h1 - h0, w1 - w0, generator=g)
        return x, y
    if content == "hdr":
        return 3 * torch.rand(C, H, W, generator=g), torch.rand(C, H, W, generator=g)
    if content == "u8":
        y = torch.randint(0, 256, (C, H, W), generator=g).float() / 255
        return (y + 0.05 * torch.randn(C, H, W, generator=g)).clamp(0, 1), y
    if content == "zeros":
        return torch.zeros(C, H, W), torch.zeros(C, H, W)
    raise ValueError(content)


def lattice(H: int, W: int, rows, cols, seed: int, C: int = 3) -> tuple:
    """Impulses at rows x cols, everything else 0; the render's impulse values differ from the ground truth's and from
    channel to channel.  Returns (x, y, support): support = the union of the 21 x 21 boxes around the impulses, clipped
    to the image -- where dL/dx is nonzero (a pixel of value 0 gets G * dm/dmu only, and dm/dmu is nonzero on the
    impulse's 11 x 11 box)."""
    g = torch.Generator().manual_seed(seed)
    x, y = torch.zeros(C, H, W), torch.zeros(C, H, W)
    r, c = torch.tensor(rows), torch.tensor(cols)
    R, Cc = torch.meshgrid(r, c, indexing="ij")
    for ch in range(C):
        x[ch, R, Cc] = 0.2 + 0.8 * torch.rand(R.shape, generator=g)
        y[ch, R, Cc] = 0.1 + 0.8 * torch.rand(R.shape, generator=g)
    rm, cm = torch.zeros(H, dtype=torch.bool), torch.zeros(W, dtype=torch.bool)
    for v in rows:
        rm[max(v - 2 * RADIUS, 0):v + 2 * RADIUS + 1] = True
    for v in cols:
        cm[max(v - 2 * RADIUS, 0):v + 2 * RADIUS + 1] = True
    return x, y, (rm[:, None] & cm[None, :]).expand(C, H, W)


def lattice_cases() -> dict:
    """736 x 736 = 23 x 32 with impulses at 23 i + 7 (23 is coprime to 32: every phase inside a 32 x 32 tile holds one), and
    a ragged 745 x 739 whose impulses also sit on the first and last rows and columns and the corners."""
    reg = list(range(7, 736, 23))
    rag_r = list(range(0, 745 - 21, 23)) + [744]
    rag_c = list(range(0, 739 - 21, 23)) + [738]
    return {"736x736": (736, 736, reg, reg), "745x739": (745, 739, rag_r, rag_c)}


def ratio(err: torch.Tensor, bound: torch.Tensor) -> float:
    """max err / bound; an element with bound 0 counts as ratio 0 when its error is 0 and inf otherwise."""
    err, bound = err.double(), bound.double()
    q = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                    torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    return float(q.max()) if q.numel() else 0.0
